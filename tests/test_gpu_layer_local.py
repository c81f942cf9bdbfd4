"""The network layers that k2y_conv2d cannot reach — the depthwise 3x3 conv, the 2x2 max-pool, the pixel-pair form of the
narrow 1x1 convs and the uint8 first conv — each checked against an fp64 reference computed from the engine's OWN input to
that layer, so the error a layer inherits from upstream plays no part in its bound (the network tests compare with the
oracle's chain, relative to the layer's maximum).

Every checked pass runs eagerly (set_keep_all, no graph) on a workspace and head buffers preset to a NaN sentinel, so an
element the pass leaves unwritten reads back as NaN."""
import functools

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from k210_yolo_framework_b200 import _lib, yolonet
from k210_yolo_framework_b200.weights import random_weights
from test_gpu_conv_tc import SENTINEL, _bound, _c_tc, _check_bound, _epilogue64, _run

TF32, X3, BF16 = _lib.MATH_TC_TF32, _lib.MATH_TC_3XTF32, _lib.MATH_TC_BF16X3
MODE_NAME = {TF32: "tf32", X3: "3xtf32", BF16: "bf16x3"}
NONE, LEAKY, RELU, RELU6 = 0, 1, 2, 3
U = 2.0 ** -24
BN_EPS32 = np.float32(1e-3)   # the BatchNormalization epsilon as the engine adds it
BATCH = 2

# (model_def, alpha, (H, W)).  The stride-1 depthwise convs of both backbones run on maps H/2 .. H/32 by W/2 .. W/32 and the
# stride-2 ones output H/4 .. H/32 by W/4 .. W/32, so W/32 = 5, 3, 4, 7 (and twice that one map up) put OW % 4 at 1, 3, 0, 3
# and 2 at both strides, and an odd H/32 gives the stride-1 form an odd OH.  C runs from 8 (alpha 0.25's conv_dw_1) to 1024.
NETS = [("yolo_mobilev1", 0.25, (64, 224)), ("yolo_mobilev1", 0.5, (96, 160)), ("yolo_mobilev1", 0.75, (64, 96)),
        ("yolo_mobilev1", 1.0, (96, 128)), ("yolo_mobilev2", 1.0, (96, 224)), ("yolo_mobilev2", 0.5, (160, 96))]
NET_IDS = [f"{m[5:]}-{a}-{hw[0]}x{hw[1]}" for m, a, hw in NETS]
DW_ACT = {"yolo_mobilev1": RELU, "yolo_mobilev2": RELU6}


def _act(model_def, name):
    """(activation, leaky slope) that net.cu's builders give mobilenet layer `name`."""
    if model_def == "yolo_mobilev2":
        return (NONE, 0.0) if name.endswith("_project") else (RELU6, 0.0)
    return (RELU, 0.0) if name.startswith("conv_dw_") else (LEAKY, 0.3)   # Keras LeakyReLU() default slope


def _engine(model_def, alpha, hw, batch):
    m, _ = getattr(yolonet, model_def)([hw[0], hw[1], 3], 3, 20, alpha=alpha, max_batch=batch)
    return m.engine


def _dw_layers(eng, hw):
    """(index in layers(), layer, (OH, OW)) of every depthwise conv.  The maps follow from the strides before it: every map
    a stride-2 layer of these backbones sees is even, and all depthwise convs come before the heads."""
    h, w = hw
    out = []
    for i, L in enumerate(eng.layers()):
        if L.stride == 2:
            assert h % 2 == 0 and w % 2 == 0
            h, w = h // 2, w // 2
        if L.kind == 1:
            out.append((i, L, (h, w)))
    return out


def _pair_layers(eng):
    """(index, layer) of the convs k2y_net_finalize gives a pixel-pair form: 1x1, stride 1, one plain source (in these
    backbones every 1x1 with Cin <= 32 has one), even Cin <= 32, Cout <= 128 and a multiple of 4."""
    return [(i, L) for i, L in enumerate(eng.layers()) if L.kind == 0 and L.kh == 1 and L.stride == 1 and L.cin <= 32
            and L.cin % 2 == 0 and L.cout <= 128 and L.cout % 4 == 0]


def _predict_on_sentinel(eng, x):
    """One eager pass (x: CUDA float32, or uint8 for the uint8 front end) with every activation and head element preset to
    the NaN sentinel.  Returns copies of the heads."""
    heads = eng.head_buffers   # binds: set_keep_all unbinds the engine, and the bind allocates a fresh workspace
    eng._ws.view(torch.int32).fill_(SENTINEL)
    for t in heads:
        t.view(torch.int32).fill_(SENTINEL)
    out = eng.predict_device_u8(x) if x.dtype == torch.uint8 else eng.predict_device(x)
    return [t.clone() for t in out]


@functools.lru_cache(maxsize=8)
def _net_pass(model_def, alpha, hw, math):
    """An engine with seeded random weights after one sentinel-preset pass on seeded [0, 1) pixels, and its weights."""
    eng = _engine(model_def, alpha, hw, BATCH)
    eng.set_keep_all(True)
    eng.set_use_graph(False)
    weights = random_weights(eng.expected_variables(), seed=7, detection_rich=True)
    eng.set_weights(weights)
    eng.set_math(math)
    x = np.random.default_rng(11).random((BATCH, hw[0], hw[1], 3), dtype=np.float32)
    _predict_on_sentinel(eng, torch.from_numpy(x).cuda())
    return eng, weights


# ---- folded BN in fp64, and what the engine's fp32 folding adds to a bound ----
# The engine folds on the host in fp32 (k2y_net_finalize):  inv = fl(gamma / fl(sqrt(fl(var + eps)))),
# shift = fl(beta - fl(mean * inv)).  With u = 2^-24 and first-order terms only:
#   inv:   the add errs by <= u relative, halved by the square root; the root and the division round once each:
#          |inv - scale| <= 2.5 u |scale|                                                      (counted as 3 u)
#   shift: fl(mean * inv) adds one rounding to inv's error: <= 3.5 u |mean * scale|; the subtraction rounds once more,
#          <= u |beta - mean * inv|:  |shift32 - shift| <= u |beta| + 4.5 u |mean * scale|      (counted as u and 5 u)
# The output is then off by |inv - scale| * |sum| + |shift32 - shift|, with |sum| <= S (the conv of |x| with |w|):
#   fold term = u * (3 |scale| S + |beta| + 5 |mean * scale|).
def _fold64(weights, bn):
    """(scale, shift, fold-term function of S) of BatchNormalization `bn`, in fp64 from the float32 variables."""
    p = {k: weights[bn][k].astype(np.float64) for k in ("gamma", "beta", "moving_mean", "moving_variance")}
    scale = p["gamma"] / np.sqrt(p["moving_variance"] + float(BN_EPS32))
    shift = p["beta"] - p["moving_mean"] * scale
    const = np.abs(p["beta"]) + 5 * np.abs(p["moving_mean"] * scale)
    return scale, shift, lambda S: U * (3 * np.abs(scale) * S + const)


def _fold32(weights, bn):
    """The engine's own fp32 folding of `bn`, operation for operation."""
    g, b, m, v = (weights[bn][k].astype(np.float32) for k in ("gamma", "beta", "moving_mean", "moving_variance"))
    inv = g / np.sqrt(v + BN_EPS32)
    return inv, b - m * inv


def _dw64(x, kernel, stride):
    """Depthwise 3x3 conv in fp64, NHWC, padded by one on every side (SAME at stride 1; ZeroPadding2D((1,1),(1,1)) + VALID
    at stride 2)."""
    t = F.pad(torch.as_tensor(x, dtype=torch.float64, device="cuda").permute(0, 3, 1, 2), (1, 1, 1, 1))
    wt = torch.as_tensor(kernel, dtype=torch.float64, device="cuda").permute(2, 3, 0, 1)   # (3,3,C,1) -> (C,1,3,3)
    return F.conv2d(t, wt, stride=stride, groups=x.shape[3]).permute(0, 2, 3, 1)


# ---- A. depthwise 3x3 (dwconv3x3_kernel: stride 1 with 2x4 outputs per thread, stride 2 with 1x4) ----
# Each output is 9 sequential fp32 FMAs from zero (padding taps add exact zeros), each rounding by <= u of a partial sum
# that is at most S: <= 9 u |scale| S before the epilogue.  _bound adds the epilogue's fmaf (with room to spare), the fold
# term above covers the fp32 constants.
@pytest.mark.gpu
@pytest.mark.parametrize("model_def,alpha,hw", NETS, ids=NET_IDS)
def test_depthwise_matches_fp64(model_def, alpha, hw):
    eng, weights = _net_pass(model_def, alpha, hw, BF16)
    layers = eng.layers()
    worst = 0.0
    for i, L, (oh, ow) in _dw_layers(eng, hw):
        name, C = L.name.decode(), L.cin
        x = eng.read_layer(layers[i - 1].name.decode(), BATCH)   # the preceding conv feeds it
        assert x.shape == (BATCH, oh * L.stride, ow * L.stride, C), name
        got = eng.read_layer(name, BATCH)
        assert got.shape == (BATCH, oh, ow, C), name
        k = weights[name]["depthwise_kernel"]
        scale, shift, fold = _fold64(weights, L.bn_name.decode())
        act, _ = _act(model_def, name)
        assert act == DW_ACT[model_def]
        ref = _epilogue64(_dw64(x, k, L.stride), scale, shift, act, 0.0, None).cpu().numpy()
        S = _dw64(np.abs(x), np.abs(k), L.stride)
        bound = _bound(S, scale, shift, None, 9 * U) + fold(S.cpu().numpy())
        what = f"{name} (stride {L.stride}, {oh}x{ow}, C {C})"
        worst = max(worst, _check_bound(got, ref, bound, what))
    print(f"depthwise {model_def}-{alpha}: worst {worst:.2%} of the bound")


# ---- B. 2x2 max-pool (maxpool2x2_kernel), bit for bit ----
# tiny_yolo's five stride-2 pools see even maps (H and W are multiples of 32); its stride-1 pool sees H/32 x W/32, here odd,
# mixed and even, with W != H.
TINY = [(96, 160), (128, 96), (64, 128)]


def _pool64(x, stride):
    """2x2 max-pool, TF 'SAME': -inf padding at the bottom and right only."""
    t = torch.as_tensor(x, dtype=torch.float64).permute(0, 3, 1, 2)
    h, w = t.shape[2], t.shape[3]
    oh, ow = -(-h // stride), -(-w // stride)
    ph, pw = max((oh - 1) * stride + 2 - h, 0), max((ow - 1) * stride + 2 - w, 0)
    return F.max_pool2d(F.pad(t, (0, pw, 0, ph), value=float("-inf")), 2, stride).permute(0, 2, 3, 1).numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("hw", TINY, ids=[f"{h}x{w}" for h, w in TINY])
def test_maxpool_is_exact(hw):
    eng, _ = _net_pass("tiny_yolo", 1.0, hw, BF16)
    for k, stride in enumerate((2, 2, 2, 2, 2, 1)):
        sfx = f"_{k}" if k else ""
        x = eng.read_layer(f"conv2d{sfx}", BATCH)       # the k-th pool reads the k-th conv
        got = eng.read_layer(f"max_pooling2d{sfx}", BATCH)
        ref = _pool64(x, stride)
        assert got.shape == ref.shape, f"max_pooling2d{sfx}"
        if stride == 1:
            assert x.shape[1:3] == (hw[0] // 32, hw[1] // 32)
        # a window whose four inputs are all negative has a negative maximum: a pool that started from 0 would miss it
        assert (ref < 0).any(), f"max_pooling2d{sfx}: no all-negative window in its input"
        np.testing.assert_array_equal(got, ref.astype(np.float32), err_msg=f"max_pooling2d{sfx} (stride {stride})")


# ---- C. the pixel-pair form of a narrow 1x1 conv (Layer::tc2) ----
# [M][K] x [K][N] runs as [M/2][2K] x blockdiag(W, W)[2K][2N] with duplicated scale and shift.  Its error is that of a
# 2K-deep GEMM in the effective mode (a bf16x3 request with 2K <= 32 runs as 3xTF32), and the same GEMM through k2y_conv2d
# (K <= 64: never split, so the same plan and instantiation) must give the same bits.
PAIRS = [(m, a, hw, mode) for m, a, hw in NETS for mode in (TF32, X3, BF16)]
PAIR_IDS = [f"{net}-{MODE_NAME[mode]}" for net in NET_IDS for mode in (TF32, X3, BF16)]


@pytest.mark.gpu
@pytest.mark.parametrize("model_def,alpha,hw,mode", PAIRS, ids=PAIR_IDS)
def test_pixel_pair_matches_fp64_and_the_pair_gemm(model_def, alpha, hw, mode):
    eng, weights = _net_pass(model_def, alpha, hw, mode)
    layers = eng.layers()
    pairs = _pair_layers(eng)
    assert pairs
    worst = 0.0
    for i, L in pairs:
        name, K, N = L.name.decode(), L.cin, L.cout
        # none of them adds a residual: the projections that do (stride 1, width kept) all have Cin >= 48
        assert not name.endswith("_project") or name == "expanded_conv_project", name
        x = eng.read_layer(layers[i - 1].name.decode(), BATCH)
        got = eng.read_layer(name, BATCH)
        assert x.shape[3] == K and got.shape == x.shape[:3] + (N,), name
        w = weights[name]["kernel"].reshape(K, N)
        act, slope = _act(model_def, name)
        scale, shift, fold = _fold64(weights, L.bn_name.decode())
        xd = torch.as_tensor(x.reshape(-1, K), dtype=torch.float64, device="cuda")
        wd = torch.as_tensor(w, dtype=torch.float64, device="cuda")
        ref = _epilogue64(xd @ wd, scale, shift, act, slope, None).cpu().numpy().reshape(got.shape)
        S = (xd.abs() @ wd.abs()).reshape(got.shape)
        eff = X3 if mode == BF16 and 2 * K <= 32 else mode
        bound = _bound(S, scale, shift, None, _c_tc(eff, 2 * K)) + fold(S.cpu().numpy())
        what = f"{name} (pair K {2 * K}, N {2 * N}, {MODE_NAME[eff]})"
        worst = max(worst, _check_bound(got, ref, bound, what))
        # the pair GEMM itself through k2y_conv2d: pixel pairs as rows, blockdiag(W, W), the engine's fp32 constants twice
        blk = np.zeros((2 * K, 2 * N), np.float32)
        blk[:K, :N] = blk[K:, N:] = w
        sc32, sh32 = _fold32(weights, L.bn_name.decode())
        M = x.shape[0] * x.shape[1] * x.shape[2]
        pair = _run(np.ascontiguousarray(x.reshape(1, 1, M // 2, 2 * K)), None, None, blk.reshape(1, 1, 2 * K, 2 * N),
                    np.tile(sc32, 2), np.tile(sh32, 2), 0, 1, 1, 0, act, slope, mode)
        assert np.array_equal(got.view(np.uint32), pair.reshape(got.shape).view(np.uint32)), \
            f"{what}: differs from the pair GEMM through k2y_conv2d"
    print(f"pixel pair {model_def}-{alpha} {MODE_NAME[mode]}: worst {worst:.2%} of the bound")


# ---- D. the uint8 first conv (first_conv3x3_kernel<N, true, ACT>) ----
# Every instantiation a net reaches: <16, leaky> (mobilev1 0.5, tiny_yolo), <24, leaky> (mobilev1 0.75), <32, leaky>
# (mobilev1 1.0, yolo), <32, relu6> (mobilev2).  Per-image output pixel counts are multiples of 128 at every input size, so
# a CTA covers one image and reads the first half of its look-up table.
U8_NETS = [("yolo_mobilev1", 0.5, (64, 96)), ("yolo_mobilev1", 0.75, (64, 64)), ("yolo_mobilev1", 1.0, (64, 96)),
           ("yolo_mobilev2", 1.0, (96, 64)), ("tiny_yolo", 1.0, (64, 96)), ("yolo", 1.0, (64, 64))]
U8_MAXIMA = (255, 127, 1, 200)   # neighbours differ, so a table built from another image's maximum shows


def _first_conv_form(model_def, L):
    return L.cout, (RELU6 if model_def == "yolo_mobilev2" else LEAKY)


@pytest.mark.gpu
@pytest.mark.parametrize("model_def,alpha,hw", U8_NETS, ids=[f"{m}-{a}" for m, a, _ in U8_NETS])
def test_uint8_first_conv_is_bit_identical(model_def, alpha, hw):
    """uint8 pixels through the on-GPU `img / np.max(img)` give the first layer's output and the heads bit for bit as the
    float32 pixels the reference computes on the host."""
    eng = _engine(model_def, alpha, hw, len(U8_MAXIMA))
    eng.set_keep_all(True)
    eng.set_use_graph(False)
    eng.set_weights(random_weights(eng.expected_variables(), seed=3, detection_rich=True))
    rng = np.random.default_rng(5)
    imgs = []
    for mx in U8_MAXIMA:
        im = rng.integers(0, mx + 1, (hw[0], hw[1], 3), dtype=np.uint8)
        im[rng.integers(hw[0]), rng.integers(hw[1]), rng.integers(3)] = mx
        imgs.append(im)
    u8 = np.stack(imgs)
    f32 = np.stack([(im / np.max(im)).astype(np.float32) for im in imgs])
    first = eng.layers()[0]
    assert (first.kh, first.cin) == (3, 3) and first.cout in (16, 24, 32)
    name = first.name.decode()
    heads_f = _predict_on_sentinel(eng, torch.from_numpy(f32).cuda())
    first_f = eng.read_layer(name, len(imgs))
    heads_u = _predict_on_sentinel(eng, torch.from_numpy(u8).cuda())
    first_u = eng.read_layer(name, len(imgs))
    assert np.isfinite(first_f).all() and np.isfinite(first_u).all(), f"{name}: unwritten elements"
    for b in range(len(imgs)):
        assert np.array_equal(first_u[b].view(np.uint32), first_f[b].view(np.uint32)), \
            f"{name}: image {b} (max {U8_MAXIMA[b]}) differs"
    for l, (a, b) in enumerate(zip(heads_f, heads_u)):
        assert torch.isfinite(a).all() and torch.equal(a, b), f"head {l} differs"


# ---- coverage of the cases above (no GPU: the graphs and their geometry come from k2y_net_create) ----
def test_layer_local_cases_cover():
    cells, dw_acts = set(), {}
    pair_ks, pair_layers = set(), set()
    for model_def, alpha, hw in NETS:
        eng = _engine(model_def, alpha, hw, BATCH)
        for _, L, (oh, ow) in _dw_layers(eng, hw):
            cells.add((L.stride, "OW%4", ow % 4))
            if L.stride == 1:
                cells.add((1, "OH%2", oh % 2))
            dw_acts.setdefault(DW_ACT[model_def], set()).add(L.cin)
        for _, L in _pair_layers(eng):
            pair_ks.add(L.cin)
            pair_layers.add((model_def, alpha, L.name.decode()))
    want = {(s, "OW%4", r) for s in (1, 2) for r in range(4)} | {(1, "OH%2", 0), (1, "OH%2", 1)}
    assert not want - cells, f"depthwise cells not reached: {sorted(want - cells)}"
    assert set(dw_acts) == {RELU, RELU6}
    assert min(min(c) for c in dw_acts.values()) == 8 and max(max(c) for c in dw_acts.values()) == 1024
    assert all(min(c) <= 32 and max(c) >= 960 for c in dw_acts.values())
    assert {16, 24, 32} <= pair_ks, f"pair K (Cin) reached: {sorted(pair_ks)}"
    for a in (0.5, 0.75, 1.0):
        assert ("yolo_mobilev1", a, "conv_pw_1") in pair_layers
    for a in (1.0, 0.5):
        assert {("yolo_mobilev2", a, "expanded_conv_project"), ("yolo_mobilev2", a, "block_1_expand")} <= pair_layers
    forms = set()
    for model_def, alpha, hw in U8_NETS:
        first = _engine(model_def, alpha, hw, 1).layers()[0]
        assert (first.kh, first.cin) == (3, 3)
        forms.add(_first_conv_form(model_def, first))
    assert forms == {(16, LEAKY), (24, LEAKY), (32, LEAKY), (32, RELU6)}
    assert all((hw[0] * hw[1] // (4 if m.startswith("yolo_mobile") else 1)) % 128 == 0 for m, _, hw in U8_NETS)
