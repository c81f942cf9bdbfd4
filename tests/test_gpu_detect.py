"""Fused decode + NMS kernels vs the oracles: bit-identical survivor sets, 1e-3 on values."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from k210_yolo_framework_b200 import Helper, KerasDetector, RegionDetector, _lib, ops
from oracle import decode_ref, region_c


def _oracle_keras(heads, anchors, in_hw, out_hw, classes, img_hw, obj, iou, maxk=30):
    h = decode_ref.HelperRef(anchors, in_hw, out_hw, classes)
    A = anchors.shape[1]
    out = []
    for b in range(heads[0].shape[0]):
        yp = [hd[b].reshape(hd.shape[1], hd.shape[2], A, 5 + classes) for hd in heads]
        out.append(decode_ref.detect_image(yp, h, in_hw, img_hw[b], obj, iou, maxk))
    return out


def _compare(got, ref):
    assert len(got) == len(ref)
    for g_img, r_img in zip(got, ref):
        assert [(d[0], d[1]) for d in g_img] == [(d[0], d[1]) for d in r_img]   # identical (class, box index) lists
        if r_img:
            np.testing.assert_allclose([d[2] for d in g_img], [d[2] for d in r_img], atol=1e-5)
            np.testing.assert_allclose([d[3:] for d in g_img], [d[3:] for d in r_img], rtol=1e-5, atol=1e-3)


def test_dog_golden_heads(dog_heads, voc_anchors, dog_u8, dog_golden):
    det = KerasDetector(voc_anchors, [224, 320], [7, 10, 14, 20], 20, 0.7, 0.5, max_batch=1)
    heads = [torch.from_numpy(dog_heads["l0_f32"]).cuda(), torch.from_numpy(dog_heads["l1_f32"]).cuda()]
    found = KerasDetector.to_host(*det.run(heads, dog_u8.shape[:2]))[0]
    gold = dog_golden["keras"]["detections"]
    assert [(d[0], d[1]) for d in found] == [(g[0], g[1]) for g in gold]
    np.testing.assert_allclose([d[2] for d in found], [g[2] for g in gold], atol=1e-5)
    np.testing.assert_allclose([d[3:] for d in found], [g[3:] for g in gold], atol=1e-3)
    # known answers (BASELINE.md §2)
    assert (found[0][0], found[0][1]) == (6, 53) and abs(found[0][2] - 0.815598) < 1e-3
    assert (found[1][0], found[1][1]) == (11, 765) and abs(found[1][2] - 0.996330) < 1e-3


@pytest.mark.parametrize("seed,batch,classes,out_hw,in_hw,obj,iou,sigma,shift", [
    (0, 4, 20, [7, 10, 14, 20], [224, 320], 0.7, 0.5, 2.0, 0.0),
    (1, 3, 20, [7, 10, 14, 20], [224, 320], 0.5, 0.3, 2.0, 1.0),      # many candidates per class, > 60 detections in an image
    (2, 2, 20, [13, 13, 26, 26], [416, 416], 0.6, 0.45, 2.5, 0.5),    # tiny_yolo geometry
    (3, 2, 80, [3, 3, 6, 6, 12, 12], [96, 96], 0.4, 0.5, 2.0, 1.5),   # 3 layers / 80 classes, NMS stress: cap of 30 binds
    (4, 2, 5, [2, 3, 4, 6], [64, 96], 0.999, 0.5, 1.0, 0.0),          # nothing passes
])
def test_seeded_heads_bit_identical_sets(seed, batch, classes, out_hw, in_hw, obj, iou, sigma, shift, voc_anchors):
    rng = np.random.default_rng(seed)
    out_hw2 = np.reshape(out_hw, (-1, 2))
    L = len(out_hw2)
    anchors = np.concatenate([voc_anchors, voc_anchors[:1] * 0.5], 0)[:L]
    heads = []
    for h, w in out_hw2:
        t = rng.normal(0, sigma, (batch, h, w, 3 * (5 + classes))).astype(np.float32)
        t = t.reshape(batch, h, w, 3, 5 + classes)
        t[..., 4:] += shift
        t[..., 2:4] *= 0.3
        heads.append(t.reshape(batch, h, w, -1))
    img_hw = np.array([[in_hw[0], in_hw[1]], [374, 499], [480, 640], [200, 100]], np.float32)[:batch]
    det = KerasDetector(anchors, in_hw, out_hw2, classes, obj, iou, max_per_class=30, max_batch=batch)
    dets, counts = det.run([torch.from_numpy(t).cuda() for t in heads], img_hw)
    got = KerasDetector.to_host(dets, counts)
    ref = _oracle_keras(heads, anchors, in_hw, out_hw2, classes, img_hw, obj, iou)
    _compare(got, ref)
    if seed == 3:
        assert int(counts.max()) == 30          # the cap binds
    if seed == 4:
        assert int(counts.sum()) == 0
    if seed == 1:
        assert max(len(i) for i in ref) > 60


def test_more_candidates_than_shared_memory_holds(voc_anchors):
    """One class with > 4096 candidates: the NMS kernel runs its global-memory rounds, reading keys and boxes from global
    memory and keeping the liveness bits there."""
    rng = np.random.default_rng(11)
    out_hw = np.array([[40, 40], [80, 80]])
    classes, batch = 2, 2
    heads = []
    for h, w in out_hw:
        t = rng.normal(0, 1.0, (batch, h, w, 3, 5 + classes)).astype(np.float32)
        t[..., 4:] += 2.5          # most boxes pass obj 0.5 in both classes
        t[..., 2:4] = t[..., 2:4] * 0.3 - 2.0   # small boxes: the cap of 30 is reached only after many suppressions
        heads.append(t.reshape(batch, h, w, -1))
    img_hw = np.array([[640, 640], [480, 600]], np.float32)
    det = KerasDetector(voc_anchors, [1280, 1280], out_hw, classes, 0.5, 0.4, max_per_class=30, max_batch=batch)
    dets, counts = det.run([torch.from_numpy(t).cuda() for t in heads], img_hw)
    got = KerasDetector.to_host(dets, counts)
    h = decode_ref.HelperRef(voc_anchors, [1280, 1280], out_hw, classes)
    ref = decode_ref.detect_batch_fast(heads, h, [1280, 1280], img_hw, 0.5, 0.4)
    n_cand = [(decode_ref.decode_layers([hd[0].reshape(hd.shape[1], hd.shape[2], 3, 5 + classes) for hd in heads], h,
                                        [1280, 1280], img_hw[0])[1] >= 0.5).sum(0).max()]
    assert n_cand[0] > 4096
    _compare(got, ref)


def _nms_tier(n, maxk, nbox):
    """The NMS tier detect_nms_kernel runs for a class with n candidates; cap = candidates its shared memory holds."""
    cap = min(-(-nbox // 256) * 256, 4096)
    if n <= 256 and maxk <= 64:
        return "chunked"
    if n <= cap:
        return "rounds4" if cap <= 2048 else "rounds8"
    return "global"


@pytest.mark.parametrize("tier,out_hw,n,maxk", [
    ("chunked", [[8, 8], [16, 16]], 256, 64),      # nbox 960, cap 1024
    ("rounds4", [[8, 8], [16, 16]], 256, 65),      # max_per_class > 64 sends a chunk-sized class to the rounds
    ("rounds4", [[8, 8], [16, 16]], 257, 30),
    ("rounds4", [[8, 8], [16, 16]], 257, 300),     # max_per_class does not bind
    ("rounds8", [[16, 16], [32, 32]], 2049, 30),   # nbox 3840 = cap
    ("rounds8", [[16, 16], [32, 32]], 3840, 30),
    ("global", [[20, 20], [40, 40]], 4097, 30),    # nbox 6000, cap 4096
])
def test_every_nms_tier(tier, out_hw, n, maxk, voc_anchors):
    """Exactly n candidates in one class put that class in the intended tier; its survivors equal the oracle's."""
    rng = np.random.default_rng(n * 1000 + maxk)
    classes, cls, in_hw = 3, 1, [256, 256]
    out_hw = np.array(out_hw)
    nbox = int(sum(h * w * 3 for h, w in out_hw))
    assert _nms_tier(n, maxk, nbox) == tier
    logits = np.full((nbox, classes), -8.0, np.float32)
    logits[rng.choice(nbox, n, replace=False), cls] = 4.0 + rng.uniform(0.0, 0.5, n)   # score ~0.98, distinct
    heads, off = [], 0
    for h, w in out_hw:
        t = np.empty((1, h, w, 3, 5 + classes), np.float32)
        t[..., 0:2] = rng.normal(0, 1.0, (1, h, w, 3, 2))
        t[..., 2:4] = rng.normal(0, 0.5, (1, h, w, 3, 2))
        t[..., 4] = 8.0
        t[..., 5:] = logits[off:off + h * w * 3].reshape(1, h, w, 3, classes)
        off += h * w * 3
        heads.append(t.reshape(1, h, w, -1))
    img_hw = np.array([[480, 640]], np.float32)
    hr = decode_ref.HelperRef(voc_anchors, in_hw, out_hw, classes)
    scores = decode_ref.decode_layers([hd[0].reshape(hd.shape[1], hd.shape[2], 3, 5 + classes) for hd in heads], hr, in_hw,
                                      img_hw[0])[1]
    assert list((scores >= 0.5).sum(0)) == [0, n, 0]
    det = KerasDetector(voc_anchors, in_hw, out_hw, classes, 0.5, 0.45, max_per_class=maxk, max_batch=1)
    got = KerasDetector.to_host(*det.run([torch.from_numpy(t).cuda() for t in heads], img_hw))
    ref = _oracle_keras(heads, voc_anchors, in_hw, out_hw, classes, img_hw, 0.5, 0.45, maxk)
    _compare(got, ref)
    assert 0 < len(ref[0]) < n    # boxes were suppressed


def test_operators_give_the_fused_kernel_bits(voc_anchors):
    """ops.tf_xywh_to_all + ops.correct_box give every box the fused kernel records, bit for bit."""
    rng = np.random.default_rng(7)
    in_hw, out_hw, classes = [224, 320], [[7, 10], [14, 20]], 20
    heads = [rng.normal(0.5, 2.0, (2, h, w, 3, 5 + classes)).astype(np.float32) for h, w in out_hw]
    img_hw = np.array([[374, 499], [480, 640]], np.float32)
    det = KerasDetector(voc_anchors, in_hw, out_hw, classes, 0.6, 0.5, max_batch=2)
    got = KerasDetector.to_host(*det.run([torch.from_numpy(t).cuda() for t in heads], img_hw))
    helper = Helper(None, classes, voc_anchors, [in_hw] * 2, out_hw)
    for b in range(2):
        boxes = []
        for layer, t in enumerate(heads):
            y = torch.from_numpy(t[b]).cuda()
            xy, wh = ops.tf_xywh_to_all(y[..., 0:2], y[..., 2:4], layer, helper)
            boxes.append(ops.correct_box(xy, wh, in_hw, img_hw[b]).reshape(-1, 4))
        boxes = torch.cat(boxes).cpu().numpy()     # box-index order: layer 0 first, then [row][col][anchor]
        assert len(got[b]) > 20
        for rec in got[b]:
            assert (np.array(rec[3:], np.float32).view(np.uint32) == boxes[rec[1]].view(np.uint32)).all(), rec


def test_strided_outputs_match_dense(voc_anchors):
    """k2y_detect_keras_strided: records and counts of one image adjacent inside a gather block (dist.DetectionGather)."""
    from k210_yolo_framework_b200.dist import DetectionGather
    rng = np.random.default_rng(5)
    heads = [torch.from_numpy(rng.normal(0.5, 2.0, (3, h, w, 75)).astype(np.float32)).cuda() for h, w in ((7, 10), (14, 20))]
    det = KerasDetector(voc_anchors, [224, 320], [7, 10, 14, 20], 20, 0.6, 0.5, max_batch=3)
    d0, c0 = det.run(heads, (224, 320))
    dense = KerasDetector.to_host(d0.clone(), c0.clone())
    g = DetectionGather(3, 20, 30, torch.device("cuda"), world=1, rank=0)
    dl, cl = g.local(0)
    det.run(heads, (224, 320), dets_out=dl, counts_out=cl)
    assert KerasDetector.to_host(*g.views(0)) == dense
    assert sum(len(i) for i in dense) > 20


def test_pinned_exponentials():
    """k2y_expf_eval: mode 0 is the correctly rounded float32 exp (KERAS dialect, == oracle.decode_ref.exp32), mode 1 is
    glibc's expf algorithm (REGION_C dialect, == this host's libm and oracle.region_c.expf_glibc) — bit for bit."""
    rng = np.random.default_rng(2)
    x = np.concatenate([rng.normal(0, 4, 200000), rng.uniform(-104, 89, 100000), [0.0, -0.0, 88.7, 88.73, -103.9, -104.5]]).astype(np.float32)
    xd = torch.from_numpy(x).cuda()
    y = torch.empty_like(xd)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(_lib.lib.k2y_expf_eval(0, xd.data_ptr(), y.data_ptr(), x.size, st))
    cr = y.cpu().numpy()
    assert (cr.view(np.uint32) == decode_ref.exp32(x).view(np.uint32)).all()
    _lib.check(_lib.lib.k2y_expf_eval(1, xd.data_ptr(), y.data_ptr(), x.size, st))
    gl = y.cpu().numpy()
    assert (gl.view(np.uint32) == region_c.expf_glibc(x).view(np.uint32)).all()
    libm = ctypes.CDLL("libm.so.6")
    libm.expf.restype = ctypes.c_float
    libm.expf.argtypes = [ctypes.c_float]
    sub = slice(0, 20000)
    assert (np.array([libm.expf(float(v)) for v in x[sub]], np.float32).view(np.uint32) == gl[sub].view(np.uint32)).all()


def test_ties_broken_by_index(voc_anchors):
    # identical logits everywhere -> equal scores; boxes of different cells do not overlap -> all kept, index ascending
    heads = [np.zeros((1, 7, 10, 75), np.float32), np.zeros((1, 14, 20, 75), np.float32)]
    for t in heads:
        t.reshape(1, t.shape[1], t.shape[2], 3, 25)[..., 2:4] = -3.0     # tiny boxes
        t.reshape(1, t.shape[1], t.shape[2], 3, 25)[..., 4:] = 6.0       # score ~0.995
    det = KerasDetector(voc_anchors, [224, 320], [7, 10, 14, 20], 20, 0.7, 0.5, max_batch=1)
    got = KerasDetector.to_host(*det.run([torch.from_numpy(t).cuda() for t in heads], (224, 320)))
    ref = _oracle_keras(heads, voc_anchors, [224, 320], np.reshape([7, 10, 14, 20], (-1, 2)), 20, [(224, 320)], 0.7, 0.5)
    _compare(got, ref)
    assert len(got[0]) == 20 * 30


ANCH = [0.76120044, 0.57155991, 0.6923348, 0.88535553, 0.47163042, 0.34163313]


@pytest.mark.parametrize("seed,w,h,classes,thr,nms,net,img,batch", [
    (0, 10, 7, 20, 0.3, 0.3, (320, 224), (320, 224), 3),
    (1, 20, 14, 20, 0.2, 0.45, (320, 224), (320, 224), 2),
    (3, 10, 7, 20, 0.3, 0.3, (320, 224), (499, 374), 2),
    (5, 26, 26, 4, 0.05, 0.3, (416, 416), (416, 416), 1),   # > 32 kept boxes per class -> list spill path
])
def test_region_kernel_vs_reference(seed, w, h, classes, thr, nms, net, img, batch):
    rng = np.random.default_rng(seed)
    x = rng.normal(0, 2.0, (batch, 3, 5 + classes, h, w)).astype(np.float32)
    x[:, :, 4] += 2.0
    x[:, :, 2:4] *= 0.3
    rd = RegionDetector(w, h, ANCH, classes, net[0], net[1], thr, nms, image_w=img[0], image_h=img[1], max_batch=batch)
    probs, boxes = rd.run(torch.from_numpy(x).cuda())
    probs, boxes = probs.cpu().numpy(), boxes.cpu().numpy()
    for b in range(batch):
        if region_c.ref_available():
            r = region_c.RegionLayerRef(w, h, 3 * (5 + classes), net[0], net[1], ANCH, thr, nms, image_width=img[0], image_height=img[1])
            r.run(x[b])
            rp, rb = r.probs(), r.boxes()
        else:
            _, rp, rb = region_c.region_layer_np(x[b], w, h, ANCH, thr, nms, net[0], net[1], img[0], img[1])
        assert ((probs[b] > 0) == (rp > 0)).all(), "survivor sets differ"
        np.testing.assert_allclose(probs[b], rp, atol=1e-6)
        np.testing.assert_allclose(boxes[b], rb, rtol=1e-5, atol=1e-6)


def test_region_layer_abi_dropin(dog_heads, voc_anchors, dog_golden):
    """main.c:278-324 call sequence against OUR library's region_layer_* symbols."""
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for l, (W, H) in enumerate([(10, 7), (20, 14)]):
        chw = region_c.nhwc_to_chw(dog_heads[f"l{l}_f32"][0], 3)
        r = region_c.RegionLayerRef(W, H, 75, 320, 224, voc_anchors[l].reshape(-1), 0.6, 0.3, lib_path=_lib.LIB_PATH)
        out = r.run(chw)
        gold = dog_golden["region_c"]["layers"][l]
        assert [list(t[:5]) for t in out] == [g[:5] for g in gold]
        assert abs(out[0][5] - gold[0][5]) < 1e-5
        r.close()


def test_detector_argument_errors(voc_anchors):
    with pytest.raises(ValueError):
        KerasDetector(voc_anchors, [224, 320], [7, 10], 20)           # anchors have 2 layers, out_hw 1
    det = KerasDetector(voc_anchors, [224, 320], [7, 10, 14, 20], 20, max_batch=1)
    with pytest.raises(ValueError):
        det.run([torch.zeros((1, 7, 10, 75), device="cuda"), torch.zeros((1, 14, 20, 74), device="cuda")], (224, 320))
    with pytest.raises(ValueError):
        det.run([torch.zeros((2, 7, 10, 75), device="cuda"), torch.zeros((2, 14, 20, 75), device="cuda")], (224, 320))
