"""Tensor-core (wgmma) conv kernel vs an fp64 convolution (and vs the fp32 CUDA-core kernel), one layer at a time through
the k2y_conv2d hook: the GEMM shapes the four networks produce, every (A path, math mode, tile width) instantiation of
conv_tc_kernel, persistent CTAs that walk several tiles, split-K, and the CUDA-core conv's own loader, grid and first-conv
forms.

Every call writes into a dst (and reads a residual) that has guard bands of sentinel bits on both sides.  Cases aimed at one
tensor-core instantiation assert it through the tile planner (k2y_tc_plan_budget), which describes the plan k2y_conv2d
launches for a plain 1x1 conv or a single-source, non-upsampled 3x3 conv."""
import ctypes
import functools

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from k210_yolo_framework_b200 import _lib
from k210_yolo_framework_b200._lib import check, lib

TF32, X3, BF16 = _lib.MATH_TC_TF32, _lib.MATH_TC_3XTF32, _lib.MATH_TC_BF16X3
MODE_NAME = {TF32: "tf32", X3: "3xtf32", BF16: "bf16x3"}
NONE, LEAKY, RELU, RELU6 = 0, 1, 2, 3
ACT_NAME = {NONE: "none", LEAKY: "leaky", RELU: "relu", RELU6: "relu6"}

GUARD = 64             # floats of sentinel bits on each side of dst and of the residual
SENTINEL = 0x7FBADBAD  # a NaN bit pattern that no kernel computes


def _guarded(n, fill=None):
    """[GUARD | n | GUARD] floats; returns the whole buffer and the n-float view.  The view starts 256 bytes into the
    allocation, so it keeps the 16-byte alignment the split-K reduce's float4 stores need."""
    buf = torch.empty(n + 2 * GUARD, dtype=torch.float32, device="cuda")
    buf.view(torch.int32).fill_(SENTINEL)
    inner = buf[GUARD:GUARD + n]
    if fill is None:
        inner.fill_(float("nan"))
    else:
        inner.copy_(fill.reshape(-1))
    return buf, inner


def _guards_intact(buf):
    bits = buf.view(torch.int32)
    return bool((bits[:GUARD] == SENTINEL).all()) and bool((bits[-GUARD:] == SENTINEL).all())


def _out_hw(h, w, ksize, stride, pad_mode):
    if pad_mode == 0:
        return h, w
    extra = 2 if pad_mode == 1 else 1
    return (h + extra - ksize) // stride + 1, (w + extra - ksize) // stride + 1


def _run(x0, x1, res, kernel, scale, shift, up0, ksize, stride, pad_mode, act, alpha, math):
    """One conv through k2y_conv2d.  Fails if it wrote outside dst or into the residual."""
    B = x0.shape[0]
    h, w = (x0.shape[1] * 2, x0.shape[2] * 2) if up0 else (x0.shape[1], x0.shape[2])
    c0, c1 = x0.shape[3], (x1.shape[3] if x1 is not None else 0)
    cout = kernel.shape[3]
    oh, ow = _out_hw(h, w, ksize, stride, pad_mode)
    n = B * oh * ow * cout
    d0 = torch.from_numpy(x0).cuda()
    d1 = torch.from_numpy(x1).cuda() if x1 is not None else None
    dbuf, out = _guarded(n)
    rbuf = dr = None
    if res is not None:
        res_dev = torch.from_numpy(np.ascontiguousarray(res, np.float32)).cuda().reshape(-1)
        rbuf, dr = _guarded(n, res_dev)
    k = np.ascontiguousarray(kernel, np.float32)
    sc, sh = np.ascontiguousarray(scale, np.float32), np.ascontiguousarray(shift, np.float32)
    st = torch.cuda.current_stream()
    check(lib.k2y_conv2d(d0.data_ptr(), d1.data_ptr() if d1 is not None else None, dr.data_ptr() if dr is not None else None,
                         out.data_ptr(), k.ctypes.data, sc.ctypes.data, sh.ctypes.data, B, h, w, c0, c1, int(up0), cout, ksize,
                         stride, pad_mode, act, float(alpha), math, ctypes.c_void_p(st.cuda_stream)))
    assert _guards_intact(dbuf), "the conv wrote outside dst"
    if res is not None:
        assert _guards_intact(rbuf) and torch.equal(dr, res_dev), "the conv wrote into the residual"
    return out.reshape(B, oh, ow, cout).cpu().numpy()


def _conv64(x0, x1, kernel, up0, ksize, stride, pad_mode):
    """The convolution alone (no BN, activation or residual) in fp64, NHWC, as a tensor on the GPU."""
    t0 = torch.as_tensor(x0, dtype=torch.float64, device="cuda").permute(0, 3, 1, 2)
    if up0:
        t0 = t0.repeat_interleave(2, 2).repeat_interleave(2, 3)
    x = t0 if x1 is None else torch.cat([t0, torch.as_tensor(x1, dtype=torch.float64, device="cuda").permute(0, 3, 1, 2)], 1)
    if pad_mode == 0:
        x = F.pad(x, (ksize // 2,) * 4)
    elif pad_mode == 1:
        x = F.pad(x, (1, 1, 1, 1))
    else:
        x = F.pad(x, (1, 0, 1, 0))
    wt = torch.as_tensor(kernel, dtype=torch.float64, device="cuda").permute(3, 2, 0, 1)
    return F.conv2d(x, wt, None, stride=stride).permute(0, 2, 3, 1)


def _epilogue64(raw, scale, shift, act, alpha, res):
    y = raw * torch.as_tensor(scale, dtype=torch.float64, device="cuda") + torch.as_tensor(shift, dtype=torch.float64, device="cuda")
    if act == LEAKY:
        y = torch.where(y >= 0, y, y * float(np.float32(alpha)))
    elif act == RELU:
        y = y.clamp(min=0)
    elif act == RELU6:
        y = y.clamp(0, 6)
    if res is not None:
        y = y + torch.as_tensor(res, dtype=torch.float64, device="cuda")
    return y


def _ref(x0, x1, res, kernel, scale, shift, up0, ksize, stride, pad_mode, act, alpha):
    return _epilogue64(_conv64(x0, x1, kernel, up0, ksize, stride, pad_mode), scale, shift, act, alpha, res).cpu().numpy()


# ---- per-element error bounds ----
# A conv output is act(scale[n] * sum_k x_k w_kn + shift[n]) (+ residual).  With S[m, n] = sum_k |x_k| |w_kn| (the fp64 conv
# of |x| with |w|) every scheme below errs by at most  c * |scale[n]| * S[m, n]  in the sum, plus the fp32 rounding of the
# epilogue (one fmaf, the leaky product, the residual add), which the activations (1-Lipschitz) do not enlarge:
#   bound = c * |scale| * S  +  2^-22 * (|scale| * S + |shift| + |residual|)
# c has a per-product part and an accumulation part.
#   tf32:    A enters the MMA as raw fp32, which the tensor core truncates to tf32 (10 stored mantissa bits): relative error
#            < 2^-10.  The weights were rounded to nearest tf32 on the host: <= 2^-11.  Per product 2^-10 + 2^-11 + 2^-21.
#   3xTF32:  a = hi + lo + r with hi = tf32(a), lo = tf32(a - hi): |a - hi| <= 2^-11 |a|, |r| <= 2^-11 |a - hi| <= 2^-22 |a|;
#            the same for w.  hi*hi + hi*lo + lo*hi drops lo*lo (<= 2^-22 |a w|) and the two r terms (<= 2^-22 each, to
#            first order): per product < 4 * 2^-22.
#   bf16x3:  the same with bf16 (8 significant bits): |a - hi| <= 2^-8 |a|, |r| <= 2^-16 |a|, lo*lo <= 2^-16 |a w|: per
#            product 3 * 2^-16, plus 2^-20 for the second-order terms.
# Accumulation: the tensor core adds a group of products to the fp32 accumulator and truncates the sum toward zero, losing
# < 1 ulp (2^-23 relative) per instruction; every partial sum is at most S.  The bound counts 2^-22 per 8 k of every pass
# (a 16-k bf16 MMA counts as two), i.e. twice the truncation of the 8-k tf32 instruction.  With split-K each slice starts
# from zero and its partial sums are bounded by its own share of S, so the chain is one slice long; the reduce pass then
# adds the `splits` partials in fp32: splits * 2^-23 more.
# The accumulation part grows like K * S while the per-product part is a fixed fraction of S, so at deep K (1152 and up) the
# split schemes' bound is far above their per-product error, and a dropped lo*hi product term, whose zero-mean errors grow only
# like sqrt(K) * 2^-12, could fit inside it.  The shallow cases carry that detection: the TMA matrix cases (K = 24 to 128)
# and the gather cases with Cin 16 and 32 (K = 144 and 288), where the whole bound is below 2^-11 * S and the dropped term's
# error is several times it.  The 1 % floor shows that no case's bound is loose by orders of magnitude, not that it is tight
# at deep K.
def _c_tc(mode, K, splits=1):
    kbk = 64 if mode == BF16 else 32  # k per k-block
    nkb = -(-K // kbk)
    slice_k = min(K, -(-nkb // splits) * kbk)
    groups = -(-slice_k // 8)
    if mode == TF32:
        per_product, passes = 2.0 ** -10 + 2.0 ** -11 + 2.0 ** -21, 1
    elif mode == X3:
        per_product, passes = 4 * 2.0 ** -22, 3
    else:
        per_product, passes = 3 * 2.0 ** -16 + 2.0 ** -20, 3
    return per_product + passes * groups * 2.0 ** -22 + (splits * 2.0 ** -23 if splits > 1 else 0.0)


# The CUDA-core conv accumulates each output with K sequential fp32 FMAs, each rounding to nearest (<= 2^-24 of the partial
# sum).  This bound is probabilistic, not rigorous, and holds only for ZERO-MEAN products: their rounding errors then have
# random signs and their sum stays within a few 2^-24 * S, and the bound allows 2^-21 (eight of them).  With products of one
# sign (the positive-mean data of the tensor-core cases) the errors add coherently, up to about K * 2^-24 * S, so the
# CUDA-core cases below draw zero-mean inputs or weights.
C_SIMT = 2.0 ** -21


def _bound(S, scale, shift, res, c):
    sS = S * torch.as_tensor(np.abs(scale), dtype=torch.float64, device="cuda")
    extra = torch.as_tensor(np.abs(shift), dtype=torch.float64, device="cuda") + (
        torch.as_tensor(np.abs(res), dtype=torch.float64, device="cuda") if res is not None else 0.0)
    return (c * sS + 2.0 ** -22 * (sS + extra)).cpu().numpy()


def _check_bound(got, ref, bound, what, floor=None):
    """Every element within its bound; with `floor`, the worst element must also use at least that share of its bound (a
    bound too loose to notice a dropped product term fails too).  Returns the worst share."""
    assert np.isfinite(got).all(), f"{what}: output has unwritten (NaN) elements"
    share = np.abs(got.astype(np.float64) - ref) / np.maximum(bound, 1e-30)
    i = np.unravel_index(int(share.argmax()), share.shape)
    worst = float(share[i])
    assert worst <= 1.0, f"{what}: error {abs(got[i] - ref[i]):.3e} at {i} exceeds its bound {bound[i]:.3e}"
    print(f"{what}: worst error {worst:.2%} of its bound")
    if floor is not None:
        assert worst >= floor, f"{what}: the worst error uses only {worst:.2%} of its bound"
    return worst


def _abs_conv64(x0, x1, kernel, up0, ksize, stride, pad_mode):
    return _conv64(np.abs(x0), None if x1 is None else np.abs(x1), np.abs(kernel), up0, ksize, stride, pad_mode)


# (B, H, W, C0, C1, up0, Cout, k, stride, pad_mode, act, residual)   H,W = stored size of src0
SHAPES = [
    (2, 28, 40, 96, 0, 0, 192, 1, 1, 0, 1, False),     # conv_pw_4 geometry: plain 1x1 via TMA, one n-tile
    (2, 56, 80, 24, 0, 0, 48, 1, 1, 0, 1, False),      # K = 24 < one k-block (TMA zero-fills), N = 48
    (3, 14, 20, 384, 0, 0, 384, 1, 1, 0, 1, False),    # conv_pw_7: several n-tiles, 12 k-blocks, ragged M (840 rows)
    (2, 7, 10, 768, 0, 0, 768, 1, 1, 0, 1, False),     # conv_pw_13: M = 140 (< 2 tiles)
    (2, 7, 10, 192, 0, 0, 75, 1, 1, 0, 0, False),      # head output: N = 75 (scalar epilogue, BN = 80)
    (2, 14, 20, 124, 0, 0, 24, 1, 1, 0, 0, True),      # mobilenet-v2 block_2 project: K = 124, N = 24, residual
    (2, 7, 10, 768, 0, 0, 192, 3, 1, 0, 1, False),     # head-1 3x3: gather path, K = 6912
    (2, 7, 10, 128, 384, 1, 128, 3, 1, 0, 1, False),   # head-2 3x3: upsample(128) || 384 concat
    (2, 16, 16, 64, 0, 0, 128, 3, 2, 2, 1, False),     # darknet downsample: pad((1,0),(1,0)) stride 2
    (2, 12, 12, 64, 0, 0, 64, 3, 1, 0, 1, True),       # darknet resblock 3x3 with residual add
    (2, 6, 6, 256, 512, 1, 256, 1, 1, 0, 1, False),    # make_last_layers first 1x1 on upsample || skip concat (gather, k=1)
    (1, 13, 13, 1024, 0, 0, 256, 1, 1, 0, 1, False),   # tiny_yolo 1x1 1024->256
    (2, 26, 30, 16, 0, 0, 32, 3, 1, 0, 1, False),      # tiny_yolo 3x3 16->32: two 16-channel taps per k-block, K = 144 padded to 160
    (1, 17, 19, 16, 0, 0, 48, 3, 2, 2, 1, False),      # same gather form, stride 2 with pad((1,0),(1,0)), odd extents
    (2, 19, 21, 32, 0, 0, 64, 3, 1, 0, 1, True),       # darknet 3x3 32->64 resblock: two 32-channel taps per bf16 k-block, K = 288 -> 320
    (1, 24, 20, 32, 0, 0, 64, 3, 2, 2, 1, False),      # darknet 3x3 32->64 stride 2
]


@pytest.mark.parametrize("math", [_lib.MATH_TC_3XTF32, _lib.MATH_TC_TF32, _lib.MATH_TC_BF16X3])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"s{i}" for i in range(len(SHAPES))])
def test_tc_conv_matches_reference(shape, math):
    B, H, W, C0, C1, up0, Cout, k, stride, pad_mode, act, use_res = shape
    rng = np.random.default_rng(hash(shape) % (2 ** 31))
    x0 = rng.normal(0, 1, (B, H, W, C0)).astype(np.float32)
    hh, ww = (H * 2, W * 2) if up0 else (H, W)
    x1 = rng.normal(0, 1, (B, hh, ww, C1)).astype(np.float32) if C1 else None
    kernel = (rng.normal(0, 1, (k, k, C0 + C1, Cout)) / np.sqrt(k * k * (C0 + C1))).astype(np.float32)
    scale = rng.uniform(0.5, 2.0, Cout).astype(np.float32)
    shift = rng.normal(0, 0.5, Cout).astype(np.float32)
    ref0 = _ref(x0, x1, None, kernel, scale, shift, up0, k, stride, pad_mode, act, 0.1)
    res = rng.normal(0, 1, ref0.shape).astype(np.float32) if use_res else None
    ref = _ref(x0, x1, res, kernel, scale, shift, up0, k, stride, pad_mode, act, 0.1)
    got = _run(x0, x1, res, kernel, scale, shift, up0, k, stride, pad_mode, act, 0.1, math)
    assert got.shape == ref.shape
    assert np.isfinite(got).all(), "output has unwritten (NaN) elements"
    err = np.abs(got - ref).max()
    # The tensor core rounds its fp32 accumulator toward zero once per MMA instruction (K = 8): a chain of
    # 3*K/8 (3xTF32) instructions loses up to ~2^-24 * chain * |acc|.  Measured: 2.4e-5 at K=384, 3.5e-4 at K=6912.
    chain = 3 * (k * k * (C0 + C1)) / 8
    if math == _lib.MATH_TC_3XTF32:
        tol = max(5e-5, 2.0 ** -24 * chain * float(np.abs(ref).max()))
    elif math == _lib.MATH_TC_BF16X3:
        tol = 6e-4   # (hi, mid) bf16 planes: ~2^-16 relative per product, random-walk over K
    else:
        tol = 2e-2
    assert err < tol, f"max abs err {err:.3e} (tol {tol:.3e})"
    # ... and every element within the scheme's own bound: the whole K as one chain, plus the fp32 adds of up to 8 split-K
    # partials.  bf16x3 requests on forms without whole 64-channel k-blocks per tap run as 3xTF32, whose bound is tighter.
    S = _abs_conv64(x0, x1, kernel, up0, k, stride, pad_mode)
    c = _c_tc(math, k * k * (C0 + C1)) + 8 * 2.0 ** -23
    _check_bound(got, ref, _bound(S, scale, shift, res, c), f"s{SHAPES.index(shape)}")
    simt = _run(x0, x1, res, kernel, scale, shift, up0, k, stride, pad_mode, act, 0.1, _lib.MATH_FP32_SIMT)
    assert np.abs(simt - ref).max() < 2e-5


def test_unsupported_shape_is_reported():
    x0 = np.zeros((1, 8, 8, 3), np.float32)
    kernel = np.zeros((3, 3, 3, 16), np.float32)
    with pytest.raises(_lib.K2YError):
        _run(x0, None, None, kernel, np.ones(16), np.zeros(16), 0, 3, 1, 0, 0, 0.0, _lib.MATH_TC_3XTF32)


# ---- the tile planner's view of a shape ----
def _plan(M, N, K, ksize, mode):
    """k2y_tc_plan_budget at the device's full SM count: the plan k2y_conv2d uses for a plain 1x1 conv or a single-source,
    non-upsampled 3x3 conv of this GEMM shape."""
    v = [ctypes.c_int() for _ in range(6)]
    check(lib.k2y_tc_plan_budget(M, N, K, ksize, mode, 0, *[ctypes.byref(x) for x in v]))
    p = dict(zip(("bn", "splits", "stages", "cluster", "math", "grid"), (x.value for x in v)))
    p["tiles"] = -(-M // 128) * -(-((N + 15) // 16 * 16) // p["bn"]) * p["splits"]
    return p


@pytest.fixture(scope="module")
def sms():
    """The device's SM count, after one conv through the hook: the planner uses the device's SM count only once the
    tensor-core path has been initialised on it."""
    x = np.ones((1, 4, 4, 32), np.float32)
    _run(x, None, None, np.ones((1, 1, 32, 16), np.float32), np.ones(16), np.zeros(16), 0, 1, 1, 0, 0, 0.0, TF32)
    n = torch.cuda.get_device_properties(0).multi_processor_count
    assert _plan(1 << 20, 128, 64, 1, TF32)["grid"] == n
    return n


def _layer_data(rng, B, H, W, C0, C1, up0, N, ksize, stride, pad_mode, act, use_res, mean):
    """Inputs and weights with the given mean (a positive mean makes the products and the accumulators' truncation errors
    share a sign), and folded-BN constants that spread each output column around 3 so that relu/relu6 clamp a real share.
    Returns the layer arguments, the fp64 reference and the bound's S."""
    x0 = rng.normal(mean, 1, (B, H, W, C0)).astype(np.float32)
    hh, ww = (H * 2, W * 2) if up0 else (H, W)
    x1 = rng.normal(mean, 1, (B, hh, ww, C1)).astype(np.float32) if C1 else None
    K = ksize * ksize * (C0 + C1)
    kernel = (rng.normal(mean, 1, (ksize, ksize, C0 + C1, N)) / np.sqrt(K)).astype(np.float32)
    raw = _conv64(x0, x1, kernel, up0, ksize, stride, pad_mode)
    mu = raw.mean(dim=(0, 1, 2)).cpu().numpy()
    sd = raw.std(dim=(0, 1, 2), unbiased=False).cpu().numpy() + 1e-3
    scale = (rng.choice([-1.0, 1.0], N) * rng.uniform(1.0, 3.0, N) / sd).astype(np.float32)
    shift = (-scale * mu + rng.normal(3.0, 2.0, N)).astype(np.float32)
    res = rng.normal(0, 1, tuple(raw.shape)).astype(np.float32) if use_res else None
    ref = _epilogue64(raw, scale, shift, act, 0.1, res).cpu().numpy()
    pre = (raw * torch.as_tensor(scale, dtype=torch.float64, device="cuda")).cpu().numpy() + shift
    S = _abs_conv64(x0, x1, kernel, up0, ksize, stride, pad_mode)
    return (x0, x1, res, kernel, scale, shift), ref, S, pre


# ---- A. every (A path, math mode, tile width) instantiation of conv_tc_kernel ----
PATHS = ("tma", "gather")
MODES = (TF32, X3, BF16)
MATRIX = [(p, m, bn) for p in PATHS for m in MODES for bn in range(16, 129, 16)]


def _matrix_form(path, mode, bn):
    """The layer form of one matrix case: (Cin, requested mode, ksize, stride, pad_mode, act, residual, odd N).
    TMA (plain 1x1): Cin puts the last k-block at 1, 2, 3 and 4 k-steps in turn (K mod 32 = 8, 16, 24, 0 with 32-wide
    k-blocks; K mod 64 = 16, 32, 40, 0 with bf16x3's 64-wide ones).  A 1x1 with K <= 32 asked for bf16x3 runs as 3xTF32.
    Gather (3x3): Cin 16 (tf32 k-blocks) and 32 (bf16 k-blocks) hold two taps per k-block; a bf16x3 request with Cin 96
    runs as 3xTF32."""
    i = bn // 16 - 1
    req = mode
    if path == "tma":
        cin = (80, 96, 104, 128)[i % 4] if mode == BF16 else (40, 48, 56, 64)[i % 4]
        if mode == X3 and i == 6:
            cin, req = 24, BF16
        ksize, stride, pad_mode = 1, 1, 0
    else:
        cin = {TF32: (16, 32, 64, 32), X3: (16, 32, 64, 96), BF16: (32, 64, 128, 64)}[mode][i % 4]
        if cin == 96:
            req = BF16
        ksize = 3
        stride, pad_mode = ((1, 0), (2, 2), (1, 0), (2, 1))[i % 4]
    act = (i + mode) % 4
    residual = (i + (path == "gather")) % 2 == 1
    return cin, req, ksize, stride, pad_mode, act, residual, i % 3 == 0


@functools.lru_cache(maxsize=None)
def _geometries(ksize, stride, pad_mode, lo, hi):
    """(B, H, W, M) with M = B * OH * OW in [lo, hi] and not a multiple of 128, at least 12 % apart."""
    found = {}
    for B in (1, 2, 3):
        for H in range(3, 400):
            for W in (H, H + 5):
                oh, ow = _out_hw(H, W, ksize, stride, pad_mode)
                M = B * oh * ow
                if lo <= M <= hi and M % 128 and M not in found:
                    found[M] = (B, H, W, M)
    out = []
    for M in sorted(found):
        if not out or M >= out[-1][3] * 1.12:
            out.append(found[M])
    return tuple(out)


_MATRIX_NS = tuple(range(4, 258)) + tuple(range(260, 769, 4)) + tuple(range(261, 769, 8))


@functools.lru_cache(maxsize=None)
def _matrix_case(path, mode, bn):
    """The smallest searched shape whose plan runs conv_tc_kernel<path, bn, mode>: (B, H, W, N), or None.  N is odd where
    the form asks for the scalar epilogue, else not a multiple of bn where such an N gets this tile."""
    cin, req, ksize, stride, pad_mode, *_, odd_n = _matrix_form(path, mode, bn)
    K = ksize * ksize * cin
    prefs = [lambda n: n % 2 == 1, lambda n: n % 2 == 0 and n % bn != 0]
    if not odd_n:
        prefs.reverse()
    for pref in prefs + [lambda n: True]:
        for B, H, W, M in _geometries(ksize, stride, pad_mode, 60, 6000):
            for N in _MATRIX_NS:
                if (N + 15) // 16 * 16 < bn or not pref(N):
                    continue
                p = _plan(M, N, K, ksize, req)
                if p["math"] == mode and p["bn"] == bn:
                    return B, H, W, N
    return None


def _conv_case(rng, B, H, W, cin, N, ksize, stride, pad_mode, act, use_res, mean=0.7):
    return _layer_data(rng, B, H, W, cin, 0, 0, N, ksize, stride, pad_mode, act, use_res, mean)


def test_matrix_covers_every_instantiation(sms):
    missing = [f"{p}-{MODE_NAME[m]}-bn{bn}" for p, m, bn in MATRIX if _matrix_case(p, m, bn) is None]
    assert not missing, f"no searched shape runs: {missing}"
    assert len(set(MATRIX)) == 48


@pytest.mark.parametrize("path,mode,bn", MATRIX, ids=[f"{p}-{MODE_NAME[m]}-bn{bn}" for p, m, bn in MATRIX])
def test_every_instantiation_matches_fp64(path, mode, bn, sms):
    case = _matrix_case(path, mode, bn)
    assert case is not None, f"no searched shape runs {path}-{MODE_NAME[mode]}-bn{bn}"
    B, H, W, N = case
    cin, req, ksize, stride, pad_mode, act, use_res, _ = _matrix_form(path, mode, bn)
    rng = np.random.default_rng(1000 * bn + 10 * mode + (path == "gather"))
    args, ref, S, pre = _conv_case(rng, B, H, W, cin, N, ksize, stride, pad_mode, act, use_res)
    if act == RELU6:
        assert (pre > 6).mean() > 0.02 and (pre < 0).mean() > 0.02
    K = ksize * ksize * cin
    p = _plan(B * ref.shape[1] * ref.shape[2], N, K, ksize, req)
    assert (p["math"], p["bn"]) == (mode, bn), p      # conv_tc_kernel<path == gather, bn, mode> runs this layer
    splits = p["splits"]
    got = _run(*args, 0, ksize, stride, pad_mode, act, 0.1, req)
    what = f"{path}-{MODE_NAME[mode]}-bn{bn} (B {B}, {H}x{W}, Cin {cin}, N {N}, {ACT_NAME[act]}, residual {use_res})"
    _check_bound(got, ref, _bound(S, args[4], args[5], args[2], _c_tc(mode, K, splits)), what, floor=0.01)


# ---- B. persistent CTAs: at least three tiles per CTA, so the stage ring's slot and phase carry across tiles ----
PERSIST = [(p, m, 0) for p in PATHS for m in MODES] + [("gather", X3, 7)]


@pytest.mark.parametrize("path,mode,splits", PERSIST,
                         ids=[f"{p}-{MODE_NAME[m]}" + (f"-split{s}" if s else "") for p, m, s in PERSIST])
def test_ctas_walk_several_tiles(path, mode, splits, sms, monkeypatch):
    if splits:
        monkeypatch.setenv("K2Y_TC_SPLITK", str(splits))
    if path == "tma":
        cin, N, ksize, stride, pad_mode = (96 if mode == BF16 else 48), 40, 1, 1, 0
    elif splits:
        cin, N, ksize, stride, pad_mode = 320, 20, 3, 1, 0      # K = 2880: 90 k-blocks in 7 slices of 13 (the last 12)
    else:
        cin, N, ksize, stride, pad_mode = 32, 24, 3, 2, 2
    K = ksize * ksize * cin
    for B, H, W, M in _geometries(ksize, stride, pad_mode, 2000, 200000):
        p = _plan(M, N, K, ksize, mode)
        if p["tiles"] >= 3 * p["grid"]:
            break
    else:
        pytest.fail("no searched shape has three tiles per CTA")
    assert p["grid"] == sms and p["math"] == mode and p["splits"] == max(splits, 1)
    act = (mode + splits) % 4
    rng = np.random.default_rng(7 * mode + splits)
    args, ref, S, _ = _conv_case(rng, B, H, W, cin, N, ksize, stride, pad_mode, act, mode != TF32)
    got = _run(*args, 0, ksize, stride, pad_mode, act, 0.1, mode)
    _check_bound(got, ref, _bound(S, args[4], args[5], args[2], _c_tc(mode, K, p["splits"])),
                 f"{path}-{MODE_NAME[mode]} M {M} N {N}: {p['tiles']} tiles on {p['grid']} CTAs", floor=0.01)


# ---- C. split-K at forced factors ----
SPLIT_SHAPES = [
    (2, 3, 3, 512, 0, 0, 1024, 3, 1, 0, LEAKY, True),   # Darknet stage-5 residual 3x3, K = 4608 (144 tf32 k-blocks)
    (2, 7, 10, 768, 0, 0, 192, 3, 1, 0, RELU6, True),   # head-1 3x3, K = 6912 (108 bf16 k-blocks), relu6 and a residual
    (2, 7, 10, 128, 384, 1, 128, 3, 1, 0, RELU, False),  # head-2 3x3 on upsample(128) || 384 concat, K = 4608
]


@pytest.mark.parametrize("splits", [2, 4, 7])
def test_split_k_matches_reference(splits, monkeypatch):
    """Deep-K 3x3 convs split their K range over several CTAs (raw partials to a scratch tensor + the reduce pass, which
    applies BN, activation and residual), in every math mode, at each shape where the forced factor applies."""
    monkeypatch.setenv("K2Y_TC_SPLITK", str(splits))
    ran = {m: [] for m in MODES}
    for math in MODES:
        for shape in SPLIT_SHAPES:
            B, H, W, C0, C1, up0, Cout, k, stride, pad_mode, act, use_res = shape
            K = k * k * (C0 + C1)
            nkb = -(-K // (64 if math == BF16 else 32))
            if nkb // splits < 12:
                continue
            p = _plan(B * H * W * (4 if up0 else 1), Cout, K, k, math)
            assert p["splits"] == splits and p["math"] == math, (shape, p)
            rng = np.random.default_rng(splits * 10 + math)
            (x0, x1, res, kernel, scale, shift), ref, S, pre = _layer_data(rng, B, H, W, C0, C1, up0, Cout, k, stride,
                                                                           pad_mode, act, use_res, 0.7)
            got = _run(x0, x1, res, kernel, scale, shift, up0, k, stride, pad_mode, act, 0.1, math)
            _check_bound(got, ref, _bound(S, scale, shift, res, _c_tc(math, K, splits)),
                         f"splits={splits} {MODE_NAME[math]} shape={shape}", floor=0.01)
            ran[math].append(shape)
    for math, shapes in ran.items():
        assert any(s[-1] for s in shapes), f"{MODE_NAME[math]}: no residual shape splits {splits} ways"
    if splits == 7:
        assert any(s[-2] == RELU6 for s in ran[BF16])


# ---- D. the CUDA-core conv (MATH_FP32_SIMT) through the same hook ----
# (id, C0, C1, ksize, N, stride, pad_mode, act, residual, tile rows per thread TM)
SIMT_CASES = [
    ("a6-n48", 6, 0, 3, 48, 1, 0, LEAKY, False, 4),     # scalar A loader (C0 % 4 != 0), not a first conv
    ("a6-n48", 6, 0, 3, 48, 1, 0, RELU, True, 8),
    ("a3-n48", 3, 0, 3, 48, 2, 2, RELU6, False, 4),
    ("a3-n48", 3, 0, 3, 48, 1, 0, NONE, True, 8),
    ("a4+2-n48", 4, 2, 1, 48, 1, 0, LEAKY, False, 4),   # concat with C1 % 4 != 0
    ("a32-n4", 32, 0, 3, 4, 1, 0, RELU6, True, 4),      # N far below the 64-column tile: 1 or 3 of its 16 column
    ("a32-n4", 32, 0, 3, 4, 2, 1, NONE, False, 8),      # groups hold columns
    ("a32-n12", 32, 0, 1, 12, 1, 0, LEAKY, False, 4),
    ("a32-n12", 32, 0, 3, 12, 1, 0, RELU, True, 8),
    ("a64-n75", 64, 0, 1, 75, 1, 0, NONE, False, 4),    # N % 4 != 0: scalar B loads and stores in the last tile
    ("a32-n75", 32, 0, 3, 75, 1, 0, LEAKY, True, 8),
]


def _simt_geometry(ksize, stride, pad_mode, N, tm, sms):
    """(B, H, W): launch_conv_simt uses 64-row tiles (TM = 4) when ceil(M / 128) * ceil(N / 64) < 2 * SMs, else 128-row
    tiles (TM = 8).  M is not a multiple of 128 either way."""
    gy = -(-N // 64)
    B, s = (2, 13) if tm == 4 else (1, 16)
    while True:
        oh, ow = _out_hw(s, s + 3, ksize, stride, pad_mode)
        M = B * oh * ow
        small = -(-M // 128) * gy < 2 * sms
        if M % 128 and small == (tm == 4):
            return B, s, s + 3
        assert tm == 8, "the TM = 4 start shape must be small"
        s += 1


@pytest.mark.parametrize("case", SIMT_CASES, ids=[f"{c[0]}-{ACT_NAME[c[7]]}-tm{c[9]}" for c in SIMT_CASES])
def test_simt_conv_forms(case, sms):
    name, C0, C1, k, N, stride, pad_mode, act, use_res, tm = case
    B, H, W = _simt_geometry(k, stride, pad_mode, N, tm, sms)
    rng = np.random.default_rng(len(name) * 100 + tm + act)
    (x0, x1, res, kernel, scale, shift), ref, S, _ = _layer_data(rng, B, H, W, C0, C1, 0, N, k, stride, pad_mode, act,
                                                                 use_res, 0.0)
    got = _run(x0, x1, res, kernel, scale, shift, 0, k, stride, pad_mode, act, 0.1, _lib.MATH_FP32_SIMT)
    _check_bound(got, ref, _bound(S, scale, shift, res, C_SIMT), f"{name} B {B} {H}x{W} tm {tm}")


# first_conv3x3_kernel: Cin 3 -> N in {16, 24, 32}; leaky and relu6 are compiled in, none and relu read the runtime act.
# Geometries: (B, H, W, stride, pad_mode) with a per-image pixel count that is not a multiple of 128, so 128-pixel CTAs
# straddle images and the last CTA is partial.
FIRST_GEOMS = [(3, 37, 29, 2, 1), (2, 45, 31, 2, 2), (3, 23, 19, 1, 0)]
FIRST_CASES = [(n, act, FIRST_GEOMS[i % 3]) for i, (n, act) in
               enumerate((n, a) for n in (16, 24, 32) for a in (LEAKY, RELU6, NONE, RELU))]


@pytest.mark.parametrize("N,act,geom", FIRST_CASES,
                         ids=[f"n{n}-{ACT_NAME[a]}-s{g[3]}p{g[4]}" for n, a, g in FIRST_CASES])
def test_first_conv_forms(N, act, geom):
    B, H, W, stride, pad_mode = geom
    oh, ow = _out_hw(H, W, 3, stride, pad_mode)
    assert (oh * ow) % 128
    rng = np.random.default_rng(N * 10 + act)
    x0 = rng.random((B, H, W, 3), dtype=np.float32)
    kernel = rng.normal(0, 0.3, (3, 3, 3, N)).astype(np.float32)
    scale = (rng.choice([-1.0, 1.0], N) * rng.uniform(1.0, 4.0, N)).astype(np.float32)
    shift = rng.normal(2.0, 2.0, N).astype(np.float32)
    ref = _ref(x0, None, None, kernel, scale, shift, 0, 3, stride, pad_mode, act, 0.1)
    S = _abs_conv64(x0, None, kernel, 0, 3, stride, pad_mode)
    got = _run(x0, None, None, kernel, scale, shift, 0, 3, stride, pad_mode, act, 0.1, _lib.MATH_FP32_SIMT)
    if act == RELU6:
        assert (ref == 6).mean() > 0.02 and (ref == 0).mean() > 0.02
    _check_bound(got, ref, _bound(S, scale, shift, None, C_SIMT), f"first conv N {N} {ACT_NAME[act]} {geom}")
