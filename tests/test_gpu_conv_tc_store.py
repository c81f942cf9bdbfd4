"""The staged epilogue of the plain 1x1 tensor-core conv: results leave through shared-memory chunks and TMA stores, which
clip rows >= M and columns >= N.  Checked bit for bit against the register epilogue of the same build, which a plain 1x1 conv
takes when dst is not 16-byte aligned (or N % 4 != 0), with sentinel bits on both sides of dst; split-K partials (which
always go through TMA stores on this path) against an fp64 bound."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from k210_yolo_framework_b200 import _lib
from k210_yolo_framework_b200._lib import check, lib

TF32, X3, BF16 = _lib.MATH_TC_TF32, _lib.MATH_TC_3XTF32, _lib.MATH_TC_BF16X3
MODES = (TF32, X3, BF16)
MODE_NAME = {TF32: "tf32", X3: "3xtf32", BF16: "bf16x3"}
GUARD = 64
SENTINEL = 0x7FBADBAD
LEAKY = 1


def _conv(x, res, kernel, scale, shift, math, offset):
    """1x1 conv of x [M, K] through k2y_conv2d into a dst that starts `offset` floats past a 256-byte boundary, with GUARD
    sentinel floats on each side.  Returns the output's int32 bits [M, N]."""
    M, N = x.shape[0], kernel.shape[1]
    n = M * N
    buf = torch.empty(n + 2 * GUARD + offset, dtype=torch.float32, device="cuda")
    buf.view(torch.int32).fill_(SENTINEL)
    out = buf[GUARD + offset:GUARD + offset + n]
    out.fill_(float("nan"))
    d0 = torch.from_numpy(x).cuda()
    dr = torch.from_numpy(res).cuda() if res is not None else None
    k = np.ascontiguousarray(kernel.reshape(1, 1, *kernel.shape), np.float32)
    st = torch.cuda.current_stream()
    check(lib.k2y_conv2d(d0.data_ptr(), None, dr.data_ptr() if dr is not None else None, out.data_ptr(), k.ctypes.data,
                         scale.ctypes.data, shift.ctypes.data, 1, 1, M, x.shape[1], 0, 0, N, 1, 1, 0, LEAKY, 0.1, math,
                         ctypes.c_void_p(st.cuda_stream)))
    bits = buf.view(torch.int32)
    assert bool((bits[:GUARD + offset] == SENTINEL).all()) and bool((bits[GUARD + offset + n:] == SENTINEL).all()), \
        "the conv wrote outside dst"
    got = out.view(torch.int32).reshape(M, N).cpu().numpy()
    assert np.isfinite(got.view(np.float32)).all(), "output has unwritten (NaN) elements"
    return got


def _plan(M, N, K, mode):
    v = [ctypes.c_int() for _ in range(6)]
    check(lib.k2y_tc_plan_budget(M, N, K, 1, mode, 0, *[ctypes.byref(x) for x in v]))
    return dict(zip(("bn", "splits", "stages", "cluster", "math", "grid"), (x.value for x in v)))


def _data(rng, M, K, N, use_res):
    x = rng.normal(0.3, 1, (M, K)).astype(np.float32)
    kernel = (rng.normal(0, 1, (K, N)) / np.sqrt(K)).astype(np.float32)
    scale = rng.uniform(0.5, 2.0, N).astype(np.float32)
    shift = rng.normal(0, 0.5, N).astype(np.float32)
    res = rng.normal(0, 1, (M, N)).astype(np.float32) if use_res else None
    return x, res, kernel, scale, shift


@pytest.fixture(scope="module")
def initialised():
    """One conv first: the planner uses the device's SM count once the tensor-core path is initialised on it."""
    rng = np.random.default_rng(0)
    x, _, kernel, scale, shift = _data(rng, 64, 32, 16, False)
    _conv(x, None, kernel, scale, shift, TF32, 0)
    return True


def _case(mode, bn):
    """(M, N): M not a multiple of 64, N a multiple of 4 but not of 32 (nor of bn where possible), planned at tile width bn."""
    K = 80 if mode == BF16 else 40   # two k-blocks; K > 32 keeps bf16x3
    for strict in (True, False):
        for M in (100, 300, 700, 1500, 3100, 6300, 12700):
            for N in range(4, 260, 4):
                if N % 32 == 0 or (strict and N % bn == 0):
                    continue
                p = _plan(M, N, K, mode)
                if p["math"] == mode and p["bn"] == bn and p["splits"] == 1:
                    return M, N, K
    return None


CASES = [(m, bn, r) for m in MODES for bn in range(16, 129, 16) for r in (False, True)]


@pytest.mark.parametrize("mode,bn,use_res", CASES, ids=[f"{MODE_NAME[m]}-bn{bn}" + ("-res" if r else "") for m, bn, r in CASES])
def test_staged_store_matches_register_epilogue(mode, bn, use_res, initialised):
    case = _case(mode, bn)
    assert case is not None, f"no searched shape plans {MODE_NAME[mode]} at bn {bn}"
    M, N, K = case
    assert M % 64 and N % 4 == 0 and N % 32
    args = _data(np.random.default_rng(bn * 10 + mode), M, K, N, use_res)
    staged = _conv(*args, mode, 0)      # 16-byte aligned dst: TMA stores
    direct = _conv(*args, mode, 2)      # 8-byte aligned dst: register epilogue
    assert np.array_equal(staged, direct), f"M {M} N {N} K {K}: staged and register epilogues differ"


@pytest.mark.parametrize("mode", MODES, ids=[MODE_NAME[m] for m in MODES])
@pytest.mark.parametrize("splits", [2, 3])
def test_split_k_partials_through_tma_stores(mode, splits, initialised, monkeypatch):
    monkeypatch.setenv("K2Y_TC_SPLITK", str(splits))
    M, N = 1000, 92
    K = 64 * 12 * splits if mode == BF16 else 32 * 12 * splits
    assert _plan(M, N, K, mode)["splits"] == splits
    x, res, kernel, scale, shift = _data(np.random.default_rng(splits * 10 + mode), M, K, N, True)
    got = _conv(x, res, kernel, scale, shift, mode, 0).view(np.float32).astype(np.float64)
    raw = torch.as_tensor(x, dtype=torch.float64) @ torch.as_tensor(kernel, dtype=torch.float64)
    y = raw * torch.as_tensor(scale, dtype=torch.float64) + torch.as_tensor(shift, dtype=torch.float64)
    ref = (torch.where(y >= 0, y, y * float(np.float32(0.1))) + torch.as_tensor(res, dtype=torch.float64)).numpy()
    S = (torch.as_tensor(np.abs(x), dtype=torch.float64) @ torch.as_tensor(np.abs(kernel), dtype=torch.float64)).numpy()
    # per product and accumulation error of each scheme (see test_gpu_conv_tc.py), one slice long, plus the reduce's adds
    per_product = {TF32: 2.0 ** -10 + 2.0 ** -11, X3: 4 * 2.0 ** -22, BF16: 3 * 2.0 ** -16 + 2.0 ** -20}[mode]
    passes = 1 if mode == TF32 else 3
    c = per_product + passes * (K // splits // 8) * 2.0 ** -22 + splits * 2.0 ** -23
    sS = S * np.abs(scale)
    bound = c * sS + 2.0 ** -22 * (sS + np.abs(shift) + np.abs(res))
    assert (np.abs(got - ref) <= bound).all()


@pytest.mark.parametrize("N", [74, 75])
def test_rows_without_16_byte_pitch_use_the_register_epilogue(N, initialised):
    """N % 4 != 0: the output is no legal tensor map, so the host picks the register epilogue (a TMA store would need a row
    pitch that is a multiple of 16 bytes, and the launch would fail).  It then does not matter how dst is aligned."""
    args = _data(np.random.default_rng(N), 333, 48, N, True)
    for mode in MODES:
        a = _conv(*args, mode, 0)
        b = _conv(*args, mode, 2)
        assert np.array_equal(a, b)
