"""HOTA (Luiten et al., 2020) on MOTChallenge sequences, restated in plain Python — TEST INFRASTRUCTURE ONLY.

This module defines the HOTA protocol that ``k210_yolo_framework_b200.evaluate.MotEval`` (csrc/evaluate_mot.cu) computes on
the GPU beside CLEAR and Identity: integer counts equal, float64 sums equal bit for bit.  It follows TrackEval's ``HOTA``
metric as far as it is known from TrackEval's published code, on the frames ``oracle.mot_ref.preprocess`` gives (the same
preprocessing CLEAR and Identity use); it has NOT been compared with TrackEval itself, which is not available here.

Ids.  G and T count the gt ids and tracker ids left after preprocessing; each gets its dense index by sorted id (TrackEval's
``np.unique``), gt id g and tracker id t sit at position g * T + t of the G x T association arrays.

Alphas: ``np.arange(0.05, 0.99, 0.05)``, 19 doubles (0.15000000000000002, ...).  A match counts at alpha a when its IoU S >=
alpha_a - eps, eps = 2^-52.

Per sequence
  1. Every frame, with or without gt or tracker rows: S = the IoU matrix of the kept rows (gt rows x tracker rows);
     denom = (S.sum(0)[None, :] + S.sum(1)[:, None]) - S; sim_iou = S / denom where denom > eps, else 0;
     pmc[g, t] += sim_iou in frame order; gc[g] += 1 and tc[t] += 1 for each id present in the frame.
  2. gas = pmc / ((gc + tc) - pmc).
  3. Every frame with both gt and tracker rows: score = gas[g, t] * S; rows, cols = lsap(-score) (every pair, no threshold,
     rows ascending); at each alpha the pairs with S >= alpha - eps count: TP += matched, FN += gt rows - matched, FP +=
     tracker rows - matched, LocA_sum += the frame's sum of their S (left to right in row order; the frame sums added in
     frame order), mc[a][g, t] += 1.  A frame without gt rows adds its tracker rows to every FP, one without tracker rows
     its gt rows to every FN.
  4. AssA_sum = np.sum(mc * (mc / np.maximum(1, (gc + tc) - mc))), AssRe_sum with np.maximum(1, gc), AssPr_sum with
     np.maximum(1, tc), each over the dense G x T array.
  5. AssX = AssX_sum / max(1, TP); LocA = max(1e-10, LocA_sum) / max(1e-10, TP); DetRe = TP / max(1, TP + FN), DetPr = TP
     / max(1, TP + FP), DetA = TP / max(1, TP + FN + FP); HOTA = sqrt(DetA * AssA), OWTA = sqrt(DetRe * AssA); HOTA(0),
     LocA(0) and HOTALocA(0) = HOTA(0) * LocA(0) at the first alpha.  TrackEval returns early for a sequence without
     tracker rows or without gt rows; these formulas give the same fields there (FN or FP = the rows, LocA = 1, the rest 0).
Combined over sequences (TrackEval's ``combine_sequences``): TP, FN and FP summed; AssA, AssRe and AssPr = sum(seq_value *
seq_TP) / max(1, TP), summed in sequence order; LocA = max(1e-10, sum(seq_LocA * seq_TP)) / max(1e-10, TP) with each
sequence's final LocA; then the final fields again.

Summation order (numpy 2.x, checked by the tests against numpy itself): ``np.sum`` of a C-contiguous float64 array (1-D, or
2-D with axis=None) is 0.0 + numpy's pairwise sum of the flattened array: fewer than 8 elements are added in order; up to
128 go into eight interleaved accumulators combined as ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)), the remainder
added in order after them; a longer array is split at n / 2 rounded down to a multiple of 8.  ``S.sum(1)`` is that sum per
row; ``S.sum(0)`` adds each column down the rows in order.  Exact zeros are neutral in that tree (every value here is >= 0),
so step 4 runs over the non-zero (g, t) entries at their dense positions (``pairwise_sum`` with `positions`).

Isolated positives.  A pair that counts at some alpha has a positive score: S >= 0.05 - eps makes denom >= S > eps (the
row and column sums each hold S, and rounding is monotone), so sim_iou > 0, pmc[g, t] > 0 and gas[g, t] > 0 (its
denominator is at least max(gc, tc) >= 1, since sim_iou <= 1).  A zero-score pair can therefore never reach alpha - eps,
whichever pairs the assignment adds.  In a frame whose positive-score entries share no row and no column, every optimal
assignment of -score takes all of them (leaving one out loses its score and gains nothing), so the pairs that count are
the positive entries with S >= alpha - eps, without an assignment.  ``hota`` uses this with ``shortcut=True``; the tests
compare it with the full assignment.

``evaluate_hota_literal`` is the same protocol written from TrackEval's code with numpy and scipy: dense matrices, masked
per-frame arrays, ``scipy.optimize.linear_sum_assignment`` and ``np.sum``.  The restatement is checked against it.
"""
from __future__ import annotations

import math
from typing import Dict, List, Sequence

import numpy as np

from oracle import mot_ref
from oracle.sort_ref import lsap

EPS = mot_ref.EPS
ALPHAS = np.arange(0.05, 0.99, 0.05).tolist()
N_ALPHA = len(ALPHAS)
ARRAY_FIELDS = ("HOTA", "DetA", "AssA", "DetRe", "DetPr", "AssRe", "AssPr", "LocA", "OWTA", "HOTA_TP", "HOTA_FN", "HOTA_FP")
SCALAR_FIELDS = ("HOTA(0)", "LocA(0)", "HOTALocA(0)")


# -- numpy's summation order ----------------------------------------------------------------------------------------------------
def _pw(vals, pos, lo: int, n: int, k0: int, k1: int) -> float:
    """Numpy's pairwise sum of the dense range [lo, lo + n), whose non-zero values are vals[k0:k1] at pos[k0:k1]."""
    if k0 == k1:
        return 0.0
    if n > 128:
        n2 = n // 2
        n2 -= n2 % 8
        km = k0
        while km < k1 and pos[km] < lo + n2:
            km += 1
        return _pw(vals, pos, lo, n2, k0, km) + _pw(vals, pos, lo + n2, n - n2, km, k1)
    nb = n - n % 8
    r = [0.0] * 8
    res = None
    for k in range(k0, k1):
        d = pos[k] - lo
        if d < nb:
            r[d % 8] += vals[k]
            continue
        if res is None:
            res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        res += vals[k]
    if res is None:
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
    return res


def pairwise_sum(values, n: int = None, positions=None) -> float:
    """``np.sum`` of a C-contiguous float64 array of values >= 0: of `values` itself, or with `positions` (ascending) of an
    array of length n holding values[k] at positions[k] and zeros elsewhere."""
    values = [float(v) for v in values]
    if positions is None:
        positions, n = list(range(len(values))), len(values)
    return 0.0 + _pw(values, [int(p) for p in positions], 0, int(n), 0, len(values))


def column_sums(S) -> list:
    """``S.sum(0)``: each column added down the rows in order."""
    out = [0.0] * (len(S[0]) if S else 0)
    for row in S:
        for j, v in enumerate(row):
            out[j] += v
    return out


# -- the restatement ------------------------------------------------------------------------------------------------------------
def counted_pairs(score, S, shortcut: bool = True) -> list:
    """The (row, col) pairs of lsap(-score), rows ascending, that have a positive score (the only ones that can count at any
    alpha); with `shortcut`, the positive entries directly when they share no row and no column."""
    if shortcut and mot_ref.isolated(score):
        return [(i, j) for i, r in enumerate(score) for j, v in enumerate(r) if v > 0]
    rows, cols = lsap([[-v for v in r] for r in score])
    return [(i, j) for i, j in zip(rows.tolist(), cols.tolist()) if score[i][j] > 0]


def final_fields(TP, FN, FP, ass_a, ass_re, ass_pr, loc_a) -> dict:
    """TrackEval's _compute_final_fields on arrays of 19."""
    TP, FN, FP = (np.asarray(x, np.float64) for x in (TP, FN, FP))
    d = dict(AssA=np.asarray(ass_a, np.float64), AssRe=np.asarray(ass_re, np.float64), AssPr=np.asarray(ass_pr, np.float64),
             LocA=np.asarray(loc_a, np.float64))
    d["DetRe"] = TP / np.maximum(1, TP + FN)
    d["DetPr"] = TP / np.maximum(1, TP + FP)
    d["DetA"] = TP / np.maximum(1, TP + FN + FP)
    d["HOTA"] = np.sqrt(d["DetA"] * d["AssA"])
    d["OWTA"] = np.sqrt(d["DetRe"] * d["AssA"])
    out = {k: [float(v) for v in d[k]] for k in ARRAY_FIELDS if k in d}
    for k, x in (("HOTA_TP", TP), ("HOTA_FN", FN), ("HOTA_FP", FP)):
        out[k] = [int(v) for v in x]
    out["HOTA(0)"] = float(d["HOTA"][0])
    out["LocA(0)"] = float(d["LocA"][0])
    out["HOTALocA(0)"] = float(d["HOTA"][0] * d["LocA"][0])
    return {k: out[k] for k in ARRAY_FIELDS + SCALAR_FIELDS}


def hota_sums(frames: Sequence[mot_ref.Frame], shortcut: bool = True) -> dict:
    """The integer counts TP / FN / FP and the float64 sums LocA / AssA / AssRe / AssPr per alpha (lists of 19), before the
    divisions of step 5."""
    thr = [a - EPS for a in ALPHAS]
    ug = sorted({g for fr in frames for g in fr.gids})
    ut = sorted({t for fr in frames for t in fr.tids})
    gi, ti = {g: k for k, g in enumerate(ug)}, {t: k for k, t in enumerate(ut)}
    T = len(ut)
    gc, tc = [0] * len(ug), [0] * T
    pmc: Dict[tuple, float] = {}
    for fr in frames:
        rs = [pairwise_sum(r) for r in fr.S]
        cs = column_sums(fr.S)
        for i, g in enumerate(fr.gids):
            for j, t in enumerate(fr.tids):
                s = fr.S[i][j]
                den = (cs[j] + rs[i]) - s
                key = (gi[g], ti[t])
                pmc[key] = pmc.get(key, 0.0) + (s / den if den > EPS else 0.0)
        for g in fr.gids:
            gc[gi[g]] += 1
        for t in fr.tids:
            tc[ti[t]] += 1
    gas = {k: v / ((gc[k[0]] + tc[k[1]]) - v) for k, v in pmc.items()}
    TP, FN, FP, loc = [0] * N_ALPHA, [0] * N_ALPHA, [0] * N_ALPHA, [0.0] * N_ALPHA
    mc: List[Dict[tuple, int]] = [{} for _ in range(N_ALPHA)]
    for fr in frames:
        ng, nt = len(fr.gids), len(fr.tids)
        if ng == 0 or nt == 0:
            for a in range(N_ALPHA):
                FP[a] += nt if ng == 0 else 0
                FN[a] += ng if nt == 0 else 0
            continue
        score = [[gas[(gi[g], ti[t])] * s for t, s in zip(fr.tids, row)] for g, row in zip(fr.gids, fr.S)]
        pairs = counted_pairs(score, fr.S, shortcut)
        for a in range(N_ALPHA):
            m = [(i, j) for i, j in pairs if fr.S[i][j] >= thr[a]]
            TP[a] += len(m)
            FN[a] += ng - len(m)
            FP[a] += nt - len(m)
            s = 0.0
            for i, j in m:
                s += fr.S[i][j]
                key = (gi[fr.gids[i]], ti[fr.tids[j]])
                mc[a][key] = mc[a].get(key, 0) + 1
            loc[a] += s
    n = len(ug) * T
    sums = {"LocA": loc, "AssA": [], "AssRe": [], "AssPr": []}
    for a in range(N_ALPHA):
        keys = sorted(mc[a], key=lambda k: k[0] * T + k[1])
        pos = [k[0] * T + k[1] for k in keys]
        m = [float(mc[a][k]) for k in keys]
        for name, den in (("AssA", lambda k, c: max(1.0, (gc[k[0]] + tc[k[1]]) - c)), ("AssRe", lambda k, c: max(1.0, gc[k[0]])),
                          ("AssPr", lambda k, c: max(1.0, tc[k[1]]))):
            sums[name].append(pairwise_sum([c * (c / den(k, c)) for k, c in zip(keys, m)], n, pos))
    return dict(HOTA_TP=TP, HOTA_FN=FN, HOTA_FP=FP, **sums)


def finish_sums(s: dict) -> dict:
    """Step 5: the per-sequence fields of ``hota_sums``."""
    TP = np.asarray(s["HOTA_TP"], np.float64)
    ass = {k: np.asarray(s[k], np.float64) / np.maximum(1, TP) for k in ("AssA", "AssRe", "AssPr")}
    loc_a = np.maximum(1e-10, np.asarray(s["LocA"], np.float64)) / np.maximum(1e-10, TP)
    return final_fields(s["HOTA_TP"], s["HOTA_FN"], s["HOTA_FP"], ass["AssA"], ass["AssRe"], ass["AssPr"], loc_a)


def hota(frames: Sequence[mot_ref.Frame], shortcut: bool = True) -> dict:
    """Every HOTA field of one sequence's preprocessed frames: lists of 19 (ARRAY_FIELDS) and the three (0) scalars."""
    return finish_sums(hota_sums(frames, shortcut))


def evaluate_hota(name: str, gt, trk, seq_length: int, benchmark: str = "MOT17", shortcut: bool = True) -> dict:
    """``hota`` of one sequence's gt and tracker rows, with mot_ref's refusals and preprocessing."""
    mot_ref.check_rows(name, gt, trk, seq_length, benchmark)
    return hota(mot_ref.preprocess(gt, trk, seq_length, benchmark), shortcut)


def combine_hota(results: Sequence[dict]) -> dict:
    """TrackEval's combine_sequences over per-sequence HOTA dicts, in sequence order."""
    TP, FN, FP = (sum(np.asarray(r[k], np.int64) for r in results) for k in ("HOTA_TP", "HOTA_FN", "HOTA_FP"))
    w = {}
    for k in ("AssRe", "AssPr", "AssA"):
        w[k] = sum(np.asarray(r[k], np.float64) * np.asarray(r["HOTA_TP"], np.float64) for r in results) / np.maximum(1.0, TP)
    loc = sum(np.asarray(r["LocA"], np.float64) * np.asarray(r["HOTA_TP"], np.float64) for r in results)
    loc_a = np.maximum(1e-10, loc) / np.maximum(1e-10, TP)
    return final_fields(TP, FN, FP, w["AssA"], w["AssRe"], w["AssPr"], loc_a)


def mean_over_alphas(d: dict) -> dict:
    """The summary TrackEval prints: each array field's mean over the alphas, and the (0) scalars."""
    out = {k: float(np.mean(d[k])) for k in ARRAY_FIELDS}
    out.update({k: d[k] for k in SCALAR_FIELDS})
    return out


# -- the literal form -----------------------------------------------------------------------------------------------------------
def _literal_frames(gt, trk, seq_length: int, benchmark: str):
    """TrackEval's preprocessing in matrix form: per frame the kept gt ids and tracker ids as sorted dense indices and the
    similarity matrix; and G, T."""
    from scipy.optimize import linear_sum_assignment
    gt, trk = np.asarray(gt, np.float64).reshape(-1, 8), np.asarray(trk, np.float64).reshape(-1, 7)
    distract = np.array(mot_ref.distractor_classes(benchmark))
    g_ids, t_ids, sims = [], [], []
    for f in range(1, seq_length + 1):
        gm, tm = gt[:, 0] == f, trk[:, 0] == f
        gi, gb, gcl, gz = gt[gm, 1].astype(int), gt[gm, 2:6], gt[gm, 7].astype(int), gt[gm, 6]
        ti, tb = trk[tm, 1].astype(int), trk[tm, 2:6]
        sim = mot_ref.box_ious(gb, tb)
        remove = np.array([], int)
        if benchmark != "MOT15" and len(gi) and len(ti):
            ms = sim.copy()
            ms[ms < 0.5 - np.finfo("float").eps] = 0
            r, c = linear_sum_assignment(-ms)
            ok = ms[r, c] > 0 + np.finfo("float").eps
            remove = c[ok][np.isin(gcl[r[ok]], distract)]
        ti, sim = np.delete(ti, remove), np.delete(sim, remove, axis=1)
        keep = (gz != 0) & (gcl == 1) if benchmark != "MOT15" else gz != 0
        g_ids.append(gi[keep])
        t_ids.append(ti)
        sims.append(sim[keep, :])
    ug = np.unique(np.concatenate(g_ids + [np.zeros(0, int)]))
    ut = np.unique(np.concatenate(t_ids + [np.zeros(0, int)]))
    return ([np.searchsorted(ug, x) for x in g_ids], [np.searchsorted(ut, x) for x in t_ids], sims, len(ug), len(ut))


def evaluate_hota_literal(gt, trk, seq_length: int, benchmark: str = "MOT17") -> dict:
    """HOTA in TrackEval's form (hota.py's eval_sequence), with numpy and scipy, written apart from the restatement."""
    from scipy.optimize import linear_sum_assignment
    eps = np.finfo("float").eps
    gt_ids, tracker_ids, sims, G, T = _literal_frames(gt, trk, seq_length, benchmark)
    alphas = np.arange(0.05, 0.99, 0.05)
    res = {k: np.zeros(len(alphas)) for k in ("HOTA_TP", "HOTA_FN", "HOTA_FP", "LocA", "AssA", "AssRe", "AssPr")}
    n_trk, n_gt = sum(len(x) for x in tracker_ids), sum(len(x) for x in gt_ids)
    if n_trk == 0 or n_gt == 0:
        res["HOTA_FN" if n_trk == 0 else "HOTA_FP"] = (n_gt if n_trk == 0 else n_trk) * np.ones(len(alphas))
        res["LocA"] = np.ones(len(alphas))
        out = {k: [float(v) for v in res[k]] for k in ("AssA", "AssRe", "AssPr", "LocA")}
        out.update({k: [0.0] * len(alphas) for k in ("HOTA", "DetA", "DetRe", "DetPr", "OWTA")})
        out.update({k: [int(v) for v in res[k]] for k in ("HOTA_TP", "HOTA_FN", "HOTA_FP")})
        out.update({"HOTA(0)": 0.0, "LocA(0)": 1.0, "HOTALocA(0)": 0.0})
        return {k: out[k] for k in ARRAY_FIELDS + SCALAR_FIELDS}
    potential_matches_count = np.zeros((G, T))
    gt_id_count = np.zeros((G, 1))
    tracker_id_count = np.zeros((1, T))
    for gt_ids_t, tracker_ids_t, similarity in zip(gt_ids, tracker_ids, sims):
        sim_iou_denom = similarity.sum(0)[np.newaxis, :] + similarity.sum(1)[:, np.newaxis] - similarity
        sim_iou = np.zeros_like(similarity)
        sim_iou_mask = sim_iou_denom > 0 + eps
        sim_iou[sim_iou_mask] = similarity[sim_iou_mask] / sim_iou_denom[sim_iou_mask]
        potential_matches_count[gt_ids_t[:, np.newaxis], tracker_ids_t[np.newaxis, :]] += sim_iou
        gt_id_count[gt_ids_t] += 1
        tracker_id_count[0, tracker_ids_t] += 1
    global_alignment_score = potential_matches_count / (gt_id_count + tracker_id_count - potential_matches_count)
    matches_counts = [np.zeros_like(potential_matches_count) for _ in alphas]
    for gt_ids_t, tracker_ids_t, similarity in zip(gt_ids, tracker_ids, sims):
        if len(gt_ids_t) == 0:
            res["HOTA_FP"] += len(tracker_ids_t)
            continue
        if len(tracker_ids_t) == 0:
            res["HOTA_FN"] += len(gt_ids_t)
            continue
        score_mat = global_alignment_score[gt_ids_t[:, np.newaxis], tracker_ids_t[np.newaxis, :]] * similarity
        match_rows, match_cols = linear_sum_assignment(-score_mat)
        for a, alpha in enumerate(alphas):
            actually_matched_mask = similarity[match_rows, match_cols] >= alpha - eps
            alpha_match_rows = match_rows[actually_matched_mask]
            alpha_match_cols = match_cols[actually_matched_mask]
            num_matches = len(alpha_match_rows)
            res["HOTA_TP"][a] += num_matches
            res["HOTA_FN"][a] += len(gt_ids_t) - num_matches
            res["HOTA_FP"][a] += len(tracker_ids_t) - num_matches
            if num_matches > 0:
                res["LocA"][a] += sum(similarity[alpha_match_rows, alpha_match_cols])
                matches_counts[a][gt_ids_t[alpha_match_rows], tracker_ids_t[alpha_match_cols]] += 1
    for a in range(len(alphas)):
        matches_count = matches_counts[a]
        ass_a = matches_count / np.maximum(1, gt_id_count + tracker_id_count - matches_count)
        res["AssA"][a] = np.sum(matches_count * ass_a) / np.maximum(1, res["HOTA_TP"][a])
        ass_re = matches_count / np.maximum(1, gt_id_count)
        res["AssRe"][a] = np.sum(matches_count * ass_re) / np.maximum(1, res["HOTA_TP"][a])
        ass_pr = matches_count / np.maximum(1, tracker_id_count)
        res["AssPr"][a] = np.sum(matches_count * ass_pr) / np.maximum(1, res["HOTA_TP"][a])
    res["LocA"] = np.maximum(1e-10, res["LocA"]) / np.maximum(1e-10, res["HOTA_TP"])
    return final_fields(res["HOTA_TP"], res["HOTA_FN"], res["HOTA_FP"], res["AssA"], res["AssRe"], res["AssPr"], res["LocA"])


def combine_hota_literal(results: Sequence[dict]) -> dict:
    """TrackEval's combine_sequences, with Python's sum over numpy arrays."""
    r = [{k: np.asarray(v, np.float64) for k, v in d.items() if k in ARRAY_FIELDS} for d in results]
    res = {k: sum(d[k] for d in r) for k in ("HOTA_TP", "HOTA_FN", "HOTA_FP")}
    for k in ("AssRe", "AssPr", "AssA"):
        res[k] = sum(d[k] * d["HOTA_TP"] for d in r) / np.maximum(1.0, res["HOTA_TP"])
    loca_weighted_sum = sum(d["LocA"] * d["HOTA_TP"] for d in r)
    res["LocA"] = np.maximum(1e-10, loca_weighted_sum) / np.maximum(1e-10, res["HOTA_TP"])
    return final_fields(res["HOTA_TP"], res["HOTA_FN"], res["HOTA_FP"], res["AssA"], res["AssRe"], res["AssPr"], res["LocA"])
