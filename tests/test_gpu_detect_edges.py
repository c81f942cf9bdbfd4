"""Fused decode + NMS at the edges of its parameters and of float32, against oracle.decode_ref (and oracle.region_c for the
REGION_C dialect): identical (class, index) lists, exact score bits, boxes to rtol 1e-6 (exactly where non-finite).

The KERAS cases are built from seeded head values whose decoded geometry was found by a search over float32 ulps with the
oracle's own decode: box pairs whose float32 IoU is exactly the threshold (kept: the test is a strict `>`), one ulp above it
(suppressed) or a few ulps either side (inside the IoU test's 1e-6 relative margin, so the exact division decides); zero-area,
infinite and NaN-area boxes from exp under/overflow; a denormal-area box inside a large one whose IoU underflows to 0; and class
and objectness logits on both sides of the exact obj_thresh boundary.  test_detect_edge_cases_cover checks on the CPU that every
NMS tier really gets them."""
import functools

import numpy as np
import pytest
import torch

from k210_yolo_framework_b200 import KerasDetector, RegionDetector, _lib, ops
from oracle import decode_ref, region_c
from test_gpu_detect import _compare, _nms_tier, _oracle_keras

f32 = np.float32
IN_HW = [256, 256]
IMG_HW = np.array([[256, 256], [300, 500]], f32)   # image 0 unletterboxed (the underflow pair needs offset 0), image 1 not
SAT, HI, MID, NEG = 20.0, 15.0, 10.0, -40.0          # sigmoid32: 1.0 exactly, 0.99999964, 0.9999546, ~4e-18


def _anchors(L, A):
    """[L, A, 2] (w, h) as fractions of the input; anchors 0 and 1 of layer 0 make the box pairs."""
    a = np.arange(A)[None, :, None]
    l = np.arange(L)[:, None, None]
    return (np.array([0.08, 0.06])[None, None] + 0.02 * a + np.array([0.0, 0.01])[None, None] * a + 0.05 * l).astype(np.float64)


# ---- float32 search helpers (the oracle's own arithmetic) ----
def _ord(x):
    b = int(np.array(x, f32).view(np.int32))
    return b if b >= 0 else -(b & 0x7FFFFFFF)


def _from_ord(k):
    k = np.asarray(k, np.int64)
    bits = np.where(k >= 0, k, (-k) | 0x80000000).astype(np.uint32)
    return bits.view(f32)


def _boundary(passes, lo, hi):
    """(first passing, last failing) float32 of a monotone predicate with passes(lo) false and passes(hi) true."""
    a, b = _ord(lo), _ord(hi)
    assert not passes(_from_ord(a)) and passes(_from_ord(b))
    while b - a > 1:
        m = (a + b) // 2
        if passes(_from_ord(m)):
            b = m
        else:
            a = m
    return float(_from_ord(b)), float(_from_ord(a))


def _cell_boxes(txy, twh, col, row, W, H, anchor, img_hw):
    """Corners of boxes at one cell for head values txy / twh [n, 2]: decode_ref.xywh_to_all's arithmetic, then correct_box."""
    xy = ((decode_ref.sigmoid32(txy) + np.array([col, row], f32)) / np.array([W, H], f32)).astype(f32)
    wh = (decode_ref.exp32(twh) * np.asarray(anchor, f32)).astype(f32)
    return decode_ref.correct_box(xy, wh, IN_HW, img_hw)


def _terms(a, b):
    """(inter, uni, iou) as decode_ref.iou_yxyx computes them, vectorised over b [n, 4]; a [4]."""
    b = np.asarray(b, f32).reshape(-1, 4)
    ya0, ya1, xa0, xa1 = min(a[0], a[2]), max(a[0], a[2]), min(a[1], a[3]), max(a[1], a[3])
    yb0, yb1 = np.minimum(b[:, 0], b[:, 2]), np.maximum(b[:, 0], b[:, 2])
    xb0, xb1 = np.minimum(b[:, 1], b[:, 3]), np.maximum(b[:, 1], b[:, 3])
    with np.errstate(all="ignore"):
        area_a = f32(f32(ya1 - ya0) * f32(xa1 - xa0))
        area_b = ((yb1 - yb0).astype(f32) * (xb1 - xb0).astype(f32)).astype(f32)
        iy = np.maximum((np.minimum(ya1, yb1) - np.maximum(ya0, yb0)).astype(f32), f32(0))
        ix = np.maximum((np.minimum(xa1, xb1) - np.maximum(xa0, xb0)).astype(f32), f32(0))
        inter = (iy * ix).astype(f32)
        uni = ((area_a + area_b).astype(f32) - inter).astype(f32)
        iou = (inter / uni).astype(f32)
    return inter, uni, np.where((area_a <= 0) | (area_b <= 0), f32(0), iou)


def _box0(col, row, W, H, anchors, tw0):
    return _cell_boxes(np.zeros((1, 2), f32), np.full((1, 2), tw0, f32), col, row, W, H, anchors[0, 0], IMG_HW[0])[0]


def _search_pair(col, row, W, H, anchors, target):
    """(tw0, tw1, th1): anchor 0 at (col, row) with tw = th = tw0 and anchor 1 with (tw1, th1) (tx = ty = 0 for both) whose
    float32 IoU is target.  The corners are pixel values, so the union moves in steps of its own ulp and the IoUs reachable
    from one first box skip some floats: the search runs over a (tw1, th1) grid and retries with another first box."""
    for k in range(40):
        tw0 = float(f32(-1.0 + 3e-4 * k))
        box0 = _box0(col, row, W, H, anchors, tw0)

        def iou(tw, th):
            twh = np.stack([np.asarray(tw, f32).ravel(), np.asarray(th, f32).ravel()], 1)
            return _terms(box0, _cell_boxes(np.zeros_like(twh), twh, col, row, W, H, anchors[0, 1], IMG_HW[0]))[2]
        tws = np.linspace(-1.6, 0.6, 4001).astype(f32)
        c = float(tws[np.argmin(np.abs(iou(tws, np.full_like(tws, -0.7)).astype(np.float64) - float(target)))]) - 0.7  # tw + th
        th = (-0.7 + np.arange(100) * 1e-5)[:, None]
        tw = c - th + (np.arange(-500, 500) * 2e-6)[None, :]
        tw, th = np.broadcast_arrays(tw.astype(f32), th.astype(f32))
        hit = np.nonzero(iou(tw, th) == f32(target))[0]
        if len(hit):
            i = hit[len(hit) // 2]
            return tw0, float(tw.ravel()[i]), float(th.ravel()[i])
    raise AssertionError(f"no pair of boxes has IoU {target!r}")


TIERS = {   # tier -> (layer sizes, max_per_class); class 0 holds nearly every box, so its candidate count puts it in the tier
    "chunked": ([[8, 8]], 64),
    "rounds4": ([[8, 8], [16, 16]], 65),      # max_per_class > 64 sends any class to the rounds
    "rounds8": ([[16, 16], [32, 32]], 65),
    "global": ([[20, 20], [40, 40]], 30),     # nbox 6000 > 4096 = cap
}
OBJS = [0.0, 1e-6, 0.5, 0.999, 1.0]
PAIR_ULPS = [0, 0, 0, 1, 1, 1, 2, -1, 3, -2, 5, -4]   # IoU - thr in float32 ulps of thr: 0 kept, > 0 suppressed, all inside 1e-6


@functools.lru_cache(maxsize=None)
def _tier_case(tier, obj):
    """Heads [2, h, w, 3 * 8] per layer (A = 3, C = 3), the pair threshold, and what each special box is (for the coverage test).
    Box index = layer offset + (row * W + col) * 3 + anchor."""
    out_hw, maxk = TIERS[tier]
    A, C = 3, 3
    anchors = _anchors(len(out_hw), A)
    H0, W0 = out_hw[0]
    heads = [np.zeros((h, w, A, 5 + C), f32) for h, w in out_hw]
    lv_special, lv_pair, lv_mass = (SAT, SAT, SAT) if obj == 1.0 else (SAT, HI, MID)
    for t in heads:                               # mass: tiny boxes at their cell centres, class 0
        t[..., 2:4] = -4.0
        t[..., 4] = SAT
        t[..., 5:] = NEG
        t[..., 5] = lv_mass
    h0 = heads[0]
    cells = iter(range(1, H0 * W0))
    info = {"pairs": [], "degenerate": [], "infinite": [], "nan_area": [], "underflow": None, "boundary": []}

    def idx(cell, a):
        return cell * A + a

    # the underflow pair: cell (0, 0), a big box at the image origin and a denormal-area box inside it
    h0[0, 0, 0, 0:5] = [-50, -50, 0, 0, SAT]
    h0[0, 0, 1, 0:5] = [-50, -50, -55, -55, SAT]
    h0[0, 0, 0:2, 5] = lv_pair
    info["underflow"] = (idx(0, 0), idx(0, 1))
    # the box pairs: anchor 0 (tw = th = -1) and anchor 1 found by the search; the first pair's IoU is the threshold
    thr = None
    for d in PAIR_ULPS:
        cell = next(cells)
        row, col = divmod(cell, W0)
        h0[row, col, 0:2, 5] = lv_pair
        if thr is None:
            thr = f32(_terms(_box0(col, row, W0, H0, anchors, -1.0), _cell_boxes(np.zeros((1, 2), f32), np.array([[-0.45, -0.7]], f32),
                                                                               col, row, W0, H0, anchors[0, 1], IMG_HW[0]))[2][0])
        tw0, tw, th = _search_pair(col, row, W0, H0, anchors, _from_ord(_ord(thr) + d))
        h0[row, col, 0, 0:4] = [0, 0, tw0, tw0]
        h0[row, col, 1, 0:4] = [0, 0, tw, th]
        info["pairs"].append((idx(cell, 0), idx(cell, 1), d))
    # special boxes ahead of everything (highest score): zero-area, infinite, infinite x zero (NaN area)
    for kind, twh in [("degenerate", (0, -110)), ("degenerate", (-110, 0)), ("infinite", (88.73, 88.73)), ("infinite", (100, 95)),
                      ("nan_area", (90, -110))]:
        cell = next(cells)
        row, col = divmod(cell, W0)
        h0[row, col, 0, 2:4] = twh
        h0[row, col, 0, 5] = lv_special
        info[kind].append(idx(cell, 0))
    # class 1: logits on both sides of the exact obj_thresh boundary (found with sigmoid32), everything else out of class 1
    sig = decode_ref.sigmoid32
    cases = []
    if obj == 0.0:
        cases = [("score 0", SAT, -110.0), ("score 0", -110.0, SAT)]
    else:
        lo = -200.0
        cls_pass, cls_fail = _boundary(lambda t: (sig(t) * sig(f32(SAT))).astype(f32) >= f32(obj), lo, 60.0)
        conf_pass, conf_fail = _boundary(lambda c: (sig(f32(SAT)) * sig(c)).astype(f32) >= f32(obj), lo, 60.0)
        cases = [("cls pass", SAT, cls_pass), ("cls fail", SAT, cls_fail), ("conf pass", conf_pass, SAT), ("conf fail", conf_fail, SAT)]
        if obj < 0.99:   # objectness sc < 1 above obj: the per-box class-logit bound is on
            for conf in (1.5, 4.0):
                sc = sig(f32(conf))
                p_, f_ = _boundary(lambda t: (sig(t) * sc).astype(f32) >= f32(obj), lo, 60.0)
                cases += [("bound pass", conf, p_), ("bound fail", conf, f_)]
    for name, conf, cls in cases:
        cell = next(cells)
        row, col = divmod(cell, W0)
        h0[row, col, 0, 4] = conf
        h0[row, col, 0, 5] = NEG
        h0[row, col, 0, 6] = cls
        info["boundary"].append((idx(cell, 0), name))
    heads = [np.ascontiguousarray(np.broadcast_to(t.reshape(1, t.shape[0], t.shape[1], -1), (2,) + t.reshape(t.shape[0], t.shape[1], -1).shape))
             for t in heads]
    return heads, anchors, out_hw, maxk, float(thr), info


def _decoded(heads, anchors, out_hw, C, b=0):
    h = decode_ref.HelperRef(anchors, IN_HW, out_hw, C)
    A = anchors.shape[1]
    return decode_ref.decode_layers([hd[b].reshape(hd.shape[1], hd.shape[2], A, 5 + C) for hd in heads], h, IN_HW, IMG_HW[b])


def _check(got, ref):
    _compare(got, ref)
    for g_img, r_img in zip(got, ref):
        for g, r in zip(g_img, r_img):
            assert np.array(g[2], f32).view(np.uint32) == np.array(r[2], f32).view(np.uint32), (g, r)
            gb, rb = np.array(g[3:], f32), np.array(r[3:], f32)
            fin = np.isfinite(rb)
            assert (gb[~fin].view(np.uint32) == rb[~fin].view(np.uint32)).all(), (g, r)
            np.testing.assert_allclose(gb[fin], rb[fin], rtol=1e-6, atol=0)


def _run_keras(heads, anchors, out_hw, C, obj, iou, maxk, img_hw=IMG_HW, strided=False):
    det = KerasDetector(anchors, IN_HW, out_hw, C, obj, iou, max_per_class=maxk, max_batch=len(img_hw))
    dev = [torch.from_numpy(np.ascontiguousarray(t)).cuda() for t in heads]
    if not strided:
        return KerasDetector.to_host(*det.run(dev, img_hw))
    n, words = len(img_hw), C * maxk * 6
    dbuf = torch.full((n, words + 40), -7, dtype=torch.int32, device="cuda")
    cbuf = torch.full((n, C + 3), -7, dtype=torch.int32, device="cuda")
    dets = torch.as_strided(dbuf, (n, C, maxk, 6), (words + 40, maxk * 6, 6, 1))
    counts = torch.as_strided(cbuf, (n, C), (C + 3, 1))
    det.run(dev, img_hw, dets_out=dets, counts_out=counts)
    out = KerasDetector.to_host(dets, counts)
    assert (dbuf[:, words:] == -7).all() and (cbuf[:, C:] == -7).all()   # nothing written between images
    return out


def _tier_n(tier, obj):
    heads, anchors, out_hw, maxk, _, _ = _tier_case(tier, obj)
    scores = _decoded(heads, anchors, out_hw, 3)[1]
    return int((scores[:, 0] >= f32(obj)).sum()), maxk, len(scores)


@pytest.mark.gpu
@pytest.mark.parametrize("obj", OBJS)
@pytest.mark.parametrize("tier", list(TIERS))
def test_tier_threshold_pairs(tier, obj):
    """Exact-threshold, one-ulp-above and in-margin pairs, degenerate / infinite / denormal boxes and obj-boundary logits,
    saturated scores tied by index; the pair threshold is the first pair's exact float32 IoU."""
    heads, anchors, out_hw, maxk, thr, _ = _tier_case(tier, obj)
    n, _, nbox = _tier_n(tier, obj)
    assert _nms_tier(n, maxk, nbox) == tier
    got = _run_keras(heads, anchors, out_hw, 3, obj, thr, maxk)
    _check(got, _oracle_keras(heads, anchors, IN_HW, out_hw, 3, IMG_HW, obj, thr, maxk))


@pytest.mark.gpu
@pytest.mark.parametrize("thr", [0.0, -0.0, -0.25], ids=["zero", "minus_zero", "negative"])
@pytest.mark.parametrize("tier", list(TIERS))
def test_tier_zero_and_negative_iou(tier, thr):
    """thr = +-0: the denormal-area box's IoU underflows to 0, so it survives its big neighbour; thr < 0: zero-area boxes
    suppress (IoU 0 > thr) and NaN IoUs (infinite boxes) do not."""
    heads, anchors, out_hw, maxk, _, info = _tier_case(tier, 0.5)
    n, _, nbox = _tier_n(tier, 0.5)
    assert _nms_tier(n, maxk, nbox) == tier
    got = _run_keras(heads, anchors, out_hw, 3, 0.5, thr, maxk)
    ref = _oracle_keras(heads, anchors, IN_HW, out_hw, 3, IMG_HW, 0.5, thr, maxk)
    _check(got, ref)
    if thr == 0.0:
        assert {info["underflow"][1]} <= {d[1] for d in ref[0] if d[0] == 0}


@pytest.mark.gpu
@pytest.mark.parametrize("thr_kind", ["pairs", "zero", "minus_zero", "negative"])
def test_operator_nms_decisions(thr_kind):
    """ops.non_max_suppression on every pair, special and underflow box of the tier cases at once: many disjoint small NMS
    problems in one call."""
    boxes, scores = [], []
    thrs = []
    for tier in TIERS:
        heads, anchors, out_hw, _, thr, info = _tier_case(tier, 0.5)
        b, s = _decoded(heads, anchors, out_hw, 3)
        sel = [i for p in info["pairs"] for i in p[:2]] + list(info["underflow"]) + info["degenerate"] + info["infinite"] + info["nan_area"]
        boxes.append(b[sel])
        scores.append(s[sel, 0] - np.arange(len(sel), dtype=f32) * f32(1e-3))   # distinct, pair member 0 first
        thrs.append(thr)
    thr = {"pairs": thrs[0], "zero": 0.0, "minus_zero": -0.0, "negative": -0.25}[thr_kind]
    if thr_kind == "pairs":   # every tier's pairs were found for its own threshold: use the first tier's boxes only
        boxes, scores = boxes[:1], scores[:1]
    boxes, scores = np.concatenate(boxes).astype(f32), np.concatenate(scores).astype(f32)
    got = ops.non_max_suppression(torch.from_numpy(boxes).cuda(), torch.from_numpy(scores).cuda(), len(boxes), thr).cpu().numpy()
    ref = decode_ref.nms_tf(boxes, scores, len(boxes), thr)
    assert got.tolist() == ref.tolist()
    assert 0 < len(ref) < len(boxes)


# ---- parameter range: C, A, layer count, max_per_class, per-image image_hw, dense and strided outputs ----
PARAMS = [   # (C, A, layer sizes, max_per_class)
    (1, 1, [[6, 5]], 1),
    (1, 5, [[4, 6], [8, 12]], 64),
    (1, 8, [[3, 4], [6, 8], [12, 16]], 65),
    (2, 8, [[2, 3], [4, 6], [8, 12]], 65),    # 3 layers x 8 anchors fill anchors[48]
    (2, 1, [[5, 5], [10, 10], [20, 20]], 1),
    (3, 5, [[4, 4], [8, 8], [16, 16]], 64),
    (3, 8, [[4, 6], [8, 12]], 65),
    (377, 1, [[4, 5], [8, 10]], 65),
    (377, 8, [[3, 4]], 1),
    (377, 5, [[2, 2], [4, 4], [8, 8]], 64),
]
PARAM_IMG_HW = np.array([[256, 256], [374, 499], [200, 100]], f32)


def _param_heads(C, A, out_hw, seed):
    rng = np.random.default_rng(seed)
    heads = []
    for h, w in out_hw:
        t = rng.normal(0, 2.0, (3, h, w, A, 5 + C)).astype(f32)
        t[..., 2:4] = t[..., 2:4] * 0.4 - 1.0
        t[..., 4] += 1.5
        t[..., 5:] += 1.0 if C <= 3 else -1.0
        heads.append(t.reshape(3, h, w, -1))
    return heads


@pytest.mark.gpu
@pytest.mark.parametrize("C,A,out_hw,maxk", PARAMS, ids=[f"C{p[0]}-A{p[1]}-L{len(p[2])}-k{p[3]}" for p in PARAMS])
def test_parameter_range(C, A, out_hw, maxk):
    heads = _param_heads(C, A, out_hw, C * 100 + A * 10 + len(out_hw))
    anchors = _anchors(len(out_hw), A)
    ref = _oracle_keras(heads, anchors, IN_HW, out_hw, C, PARAM_IMG_HW, 0.5, 0.45, maxk)
    dense = _run_keras(heads, anchors, out_hw, C, 0.5, 0.45, maxk, PARAM_IMG_HW)
    _check(dense, ref)
    assert _run_keras(heads, anchors, out_hw, C, 0.5, 0.45, maxk, PARAM_IMG_HW, strided=True) == dense
    assert all(len(i) > 0 for i in ref)
    if maxk > 1:
        assert max(len(i) for i in ref) > C   # some class keeps more than one box


@pytest.mark.gpu
def test_class_num_beyond_scan_slab_rejected():
    """C = 378: 64 boxes x (5 + C + 2) floats exceed the scan kernel's 96 KB slab."""
    anchors = _anchors(1, 3)
    det = KerasDetector(anchors, IN_HW, [[4, 4]], 378, 0.5, 0.45, max_per_class=4, max_batch=1)
    heads = [torch.zeros((1, 4, 4, 3 * (5 + 378)), device="cuda")]
    with pytest.raises(_lib.K2YError, match=r"^\[-1\]"):
        det.run(heads, (256, 256))


# ---- REGION_C dialect ----
ANCH5 = [1.08, 1.19, 3.42, 4.41, 6.63, 11.38, 9.42, 5.11, 16.62, 10.52]
REGION = [   # (C, W, H, thr, nms, image (w, h))
    (1, 16, 16, 0.3, 0.45, (320, 240)),    # N = 1280
    (80, 16, 16, 0.2, 0.4, (416, 416)),    # 80 classes: the warp-per-class loop wraps past 32 warps
    (80, 6, 7, 0.1, 0.3, (320, 224)),
]


def _region_input(C, W, H, seed):
    rng = np.random.default_rng(seed)
    x = rng.normal(0, 1.0, (2, 5, 5 + C, H, W)).astype(f32)
    x[:, :, 2:4] = x[:, :, 2:4] * 0.3 - 2.5
    x[:, :, 4] += 1.0
    if C > 1:
        dom = rng.integers(0, 3 if C > 3 else C, (2, 5, H, W))
        np.put_along_axis(x[:, :, 5:], dom[:, :, None], 6.0 + rng.uniform(0, 1, (2, 5, 1, H, W)).astype(f32), axis=2)
    # exp over- and underflow: infinite / zero widths, sigmoid exactly 0 or 1, softmax terms that underflow to 0
    x[:, 0, 2, 0, :4] = 90.0
    x[:, 1, 3, 0, :4] = -110.0
    x[:, 2, 0, 1, :3] = -110.0
    x[:, 2, 1, 1, :3] = 110.0
    x[:, 3, 4, 1, 0] = 120.0   # one box only: with one class its prob 1.0 would tie
    if C > 1:
        x[:, 4, 5, 1, :3] = 60.0
        x[:, 4, 6:, 1, :3] = -60.0
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("C,W,H,thr,nms,img", REGION, ids=[f"C{r[0]}-{r[1]}x{r[2]}" for r in REGION])
def test_region_edges(C, W, H, thr, nms, img):
    x = _region_input(C, W, H, C + W)
    rd = RegionDetector(W, H, ANCH5, C, 416, 416, thr, nms, image_w=img[0], image_h=img[1], max_batch=2)
    probs, boxes = (t.cpu().numpy() for t in rd.run(torch.from_numpy(x).cuda()))
    for b in range(2):
        if region_c.ref_available():
            r = region_c.RegionLayerRef(W, H, 5 * (5 + C), 416, 416, ANCH5, thr, nms, image_width=img[0], image_height=img[1])
            r.run(x[b])
            rp, rb = r.probs(), r.boxes()
            r.close()
        else:
            _, rp, rb = region_c.region_layer_np(x[b], W, H, ANCH5, thr, nms, 416, 416, img[0], img[1])
        cand = rp[:, :C]
        for k in range(C):   # no exact ties among a class's candidates: the reference's qsort order of ties is unspecified
            v = cand[cand[:, k] > 0, k]
            assert len(np.unique(v)) == len(v)
        assert ((probs[b] > 0) == (rp > 0)).all(), "survivor sets differ"
        np.testing.assert_allclose(probs[b], rp, rtol=1e-6, atol=0)
        np.testing.assert_allclose(boxes[b], rb, rtol=1e-6, atol=1e-7)
        assert np.isinf(rb[:, 2]).any() and (rb[:, 3] == 0).any()
        if W * H * 5 > 1024:
            assert ((probs[b][:, :C] > 0).sum(0) > 32).any()


# ---- coverage of the cases above (no GPU: the oracle decodes them on the CPU) ----
def test_detect_edge_cases_cover():
    for tier in TIERS:
        got = {"exact": 0, "above": 0, "margin": 0, "degenerate": 0, "infinite": 0}
        for obj in OBJS:
            heads, anchors, out_hw, maxk, thr, info = _tier_case(tier, obj)
            n, _, nbox = _tier_n(tier, obj)
            assert _nms_tier(n, maxk, nbox) == tier, (tier, obj, n)
            boxes, scores = _decoded(heads, anchors, out_hw, 3)
            cand = scores[:, 0] >= f32(obj)
            thr32 = f32(thr)
            for i0, i1, d in info["pairs"]:
                assert cand[i0] and cand[i1]
                q = decode_ref.iou_yxyx(boxes[i0], boxes[i1])
                assert q == _from_ord(_ord(thr32) + d), (tier, obj, d)
                assert abs(float(q) - float(thr32)) <= 1e-6 * float(thr32)
                got["exact"] += q == thr32
                got["above"] += q == np.nextafter(thr32, f32(1))
                got["margin"] += q != thr32
            with np.errstate(all="ignore"):
                areas = (np.abs(boxes[:, 2] - boxes[:, 0]) * np.abs(boxes[:, 3] - boxes[:, 1])).astype(f32)
            for i in info["degenerate"]:
                assert cand[i] and areas[i] == 0
                got["degenerate"] += 1
            for i in info["infinite"]:
                assert cand[i] and np.isinf(boxes[i]).all() and np.isinf(areas[i])
                got["infinite"] += 1
            for i in info["nan_area"]:
                assert np.isnan(areas[i])
            # the underflow pair: inter > 0, yet fl(inter / uni) == 0
            i0, i1 = info["underflow"]
            inter, uni, _ = _terms(boxes[i0], boxes[i1:i1 + 1])
            assert cand[i0] and cand[i1] and inter[0] > 0 and f32(inter[0] / uni[0]) == 0
            assert 0 < areas[i1] < np.finfo(f32).tiny   # denormal area
            assert decode_ref.iou_yxyx(boxes[i0], boxes[i1]) == 0
            # obj boundary logits: the pass / fail pairs straddle obj exactly
            s1 = scores[:, 1]
            for i, name in info["boundary"]:
                assert (s1[i] >= f32(obj)) == (name.endswith("pass") or name == "score 0"), (tier, obj, name, s1[i])
            names = {nm for _, nm in info["boundary"]}
            if 0 < obj < 0.99:
                assert {"bound pass", "bound fail", "cls pass", "cls fail", "conf pass", "conf fail"} <= names
            if obj == 0:
                assert (s1[[i for i, _ in info["boundary"]]] == 0).all()
            assert (scores[info["degenerate"] + info["infinite"], 0] == 1).all()   # saturated: ties broken by index
        assert min(got.values()) >= 1, (tier, got)
    cells = {("C", p[0]) for p in PARAMS} | {("A", p[1]) for p in PARAMS} | {("L", len(p[2])) for p in PARAMS} | \
        {("k", p[3]) for p in PARAMS}
    want = {("C", c) for c in (1, 2, 3, 377)} | {("A", a) for a in (1, 5, 8)} | {("L", l) for l in (1, 2, 3)} | \
        {("k", k) for k in (1, 64, 65)}
    assert not want - cells, sorted(want - cells)
    assert any(p[1] == 8 and len(p[2]) == 3 for p in PARAMS)
    for C, A, out_hw, _ in PARAMS:
        assert 64 * (5 + C + 2) * 4 <= 96 * 1024
    assert 64 * (5 + 378 + 2) * 4 > 96 * 1024
    assert len({tuple(r) for r in PARAM_IMG_HW}) == len(PARAM_IMG_HW)
    assert {r[0] for r in REGION} == {1, 80} and any(r[1] * r[2] * 5 > 1024 for r in REGION)


def test_scan_item_split_is_exact():
    """The scan kernel splits item `it` of a 64-box slab into (box it / C, class it % C) as (it * ceil(2^32 / C)) >> 32 with
    a 64-bit magic; a 32-bit one truncates to 0 at C = 1."""
    for C in range(1, 378):
        m = (2 ** 32 + C - 1) // C
        it = np.arange(64 * C, dtype=np.uint64)
        assert ((it * np.uint64(m)) >> np.uint64(32) == it // np.uint64(C)).all(), C
        if C > 1:   # the 32-bit magic is right for C >= 2 ...
            assert m < 2 ** 32
    it = np.arange(64, dtype=np.uint64)   # ... and wrong for 63 of the 64 items of a slab at C = 1
    assert ((it * np.uint64((2 ** 32) & 0xFFFFFFFF)) >> np.uint64(32) != it).sum() == 63
