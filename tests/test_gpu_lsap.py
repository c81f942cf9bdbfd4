"""``warp_lsap`` (csrc/lsap_warp.cuh), the assignment solver of ByteTrack, OC-SORT and the MOT evaluator, against
scipy.optimize.linear_sum_assignment: every pair equal, ties included.  The matrices are chosen for what a warp-wide
solver can get wrong: the tie key across lanes, column counts on either side of a multiple of 32, the transposed case, -0.0
beside +0.0, 512 x 512 in shared memory and a large problem in global memory.  tests/lsap_harness.cu runs one warp per
problem; it is compiled here with the library's nvcc flags and is not part of the library."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
from scipy.optimize import linear_sum_assignment

from conftest import ROOT

CSRC = os.path.join(ROOT, "k210_yolo_framework_b200", "csrc")
HARNESS = os.path.join(ROOT, "tests", "lsap_harness.cu")
SHARED_CAP = 512        # K2Y_MOT_MAX_ROWS: the shared kernel's entries per array


def _nvcc_cmd(out):
    from k210_yolo_framework_b200 import build
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    return [nvcc] + build.NVCC_FLAGS + ["-I", CSRC, "-I", os.path.join(ROOT, "include"), "-o", out, HARNESS]


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("lsap") / "lsap_harness.so")
    r = subprocess.run(_nvcc_cmd(out), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    lib = ctypes.CDLL(out)
    lib.lsap_harness_run.restype = ctypes.c_int
    lib.lsap_harness_run.argtypes = [ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 8 + [ctypes.c_longlong] + \
        [ctypes.c_void_p] * 3
    return lib


def test_harness_compiles_and_loads(harness):
    assert harness.lsap_harness_run(0, 0, *([None] * 8), 0, None, None, None) == 0


# -- cost matrices -------------------------------------------------------------------------------------------------------
def _signed_zeros(rng, shape):
    return np.where(rng.random(shape) < 0.5, -0.0, 0.0)


def _cost(kind, rng, nr, nc):
    """A float64 nr x nc matrix of one kind."""
    shape = (nr, nc)
    if kind == "uniform":
        return rng.random(shape)
    if kind == "ints":                          # small negated integers: ties at every step
        return -rng.integers(0, 3, shape).astype(np.float64)
    if kind == "equal":
        return np.full(shape, float(rng.choice([0.0, -0.0, 1.0, -2.5])))
    if kind == "dup_rows":
        base = -rng.integers(0, 4, (max(1, (nr + 2) // 3), nc)).astype(np.float64)
        return base[rng.integers(0, len(base), nr)]
    if kind == "dup_cols":
        base = rng.random((nr, max(1, (nc + 2) // 3)))
        return base[:, rng.integers(0, base.shape[1], nc)]
    if kind == "sparse_iou":                    # -IoU as the evaluator's costs: mostly zeros of either sign
        c = _signed_zeros(rng, shape)
        hit = rng.random(shape) < 0.08
        iou = np.where(rng.random(shape) < 0.3, 0.5, 0.5 + rng.integers(0, 5, shape) / 8.0)
        return np.where(hit, -iou, c)
    if kind == "clear_bonus":                   # CLEAR's -(1000 + s) for the previous frame's pairs, -s, signed zeros
        c = _signed_zeros(rng, shape)
        s = 0.5 + rng.integers(0, 5, shape) / 8.0
        r = rng.random(shape)
        return np.where(r < 0.05, -(1000.0 + s), np.where(r < 0.2, -s, c))
    if kind == "magnitudes":                    # 1e-9 .. 1e9: reduced costs ((min_val + c) - u) - v round into ties
        m = 10.0 ** rng.integers(-9, 10, shape)
        return m * rng.integers(-2, 3, shape)
    raise ValueError(kind)


KINDS = ["uniform", "ints", "equal", "dup_rows", "dup_cols", "sparse_iou", "clear_bonus", "magnitudes"]
SHAPES = [(0, 5), (5, 0), (0, 0), (1, 1), (1, 40), (40, 1), (31, 32), (32, 33), (33, 31), (63, 64), (64, 65), (65, 64),
          (7, 100), (100, 7), (2, 2), (3, 5), (32, 32), (33, 33)]
LARGE = [(512, 512), (512, 97), (97, 512)]


def _scipy(c):
    """match[i] = scipy's column of row i, -1 for a row it leaves out."""
    m = np.full(c.shape[0], -1, np.int32)
    if c.size:
        r, k = linear_sum_assignment(c)
        m[r] = k
    return m


def _solve(lib, mats, shared):
    """warp_lsap's match of every matrix, one warp each, in one launch."""
    import torch
    dev = torch.device("cuda", 0)
    nr = np.array([m.shape[0] for m in mats], np.int32)
    nc = np.array([m.shape[1] for m in mats], np.int32)
    coff = np.concatenate([[0], np.cumsum(nr.astype(np.int64) * nc)])
    moff = np.concatenate([[0], np.cumsum(nr.astype(np.int64))])
    ent = np.maximum(nr, nc).astype(np.int64)
    woff = np.concatenate([[0], np.cumsum(ent)])
    wn = int(woff[-1])
    if shared:
        assert ent.max() <= SHARED_CAP
    cost = torch.from_numpy(np.concatenate([m.ravel() for m in mats] + [np.zeros(1)])).to(dev)
    t = {k: torch.from_numpy(v).to(dev) for k, v in dict(coff=coff, moff=moff, woff=woff, nr=nr, nc=nc).items()}
    match = torch.full((int(moff[-1]) + 1,), -7, dtype=torch.int32, device=dev)
    wd = torch.empty(3 * wn + 1, dtype=torch.float64, device=dev)
    wi = torch.empty(4 * wn + 1, dtype=torch.int32, device=dev)
    wb = torch.empty(2 * wn + 1, dtype=torch.uint8, device=dev)
    st = torch.cuda.current_stream(dev)
    err = lib.lsap_harness_run(len(mats), int(shared), cost.data_ptr(), t["coff"].data_ptr(), t["nr"].data_ptr(),
                               t["nc"].data_ptr(), t["woff"].data_ptr(), wd.data_ptr(), wi.data_ptr(), wb.data_ptr(), wn,
                               match.data_ptr(), t["moff"].data_ptr(), ctypes.c_void_p(st.cuda_stream))
    assert err == 0
    torch.cuda.synchronize(dev)
    out = match.cpu().numpy()
    return [out[moff[p]:moff[p + 1]] for p in range(len(mats))]


def _check(lib, mats, shared, what, kinds=None):
    got = _solve(lib, mats, shared)
    bad = [p for p, (m, g) in enumerate(zip(mats, got)) if not np.array_equal(g, _scipy(m))]
    assert not bad, (what, len(bad), [(mats[p].shape, kinds[p] if kinds else None) for p in bad[:8]])


def _problems(seed, shapes, per):
    """(matrices, their kinds): `per` matrices of every kind at every shape."""
    rng = np.random.default_rng(seed)
    kinds = [k for k in KINDS for _ in shapes for _ in range(per)]
    return [_cost(k, rng, nr, nc) for k in KINDS for nr, nc in shapes for _ in range(per)], kinds


@pytest.mark.gpu
@pytest.mark.parametrize("shared", [1, 0], ids=["shared", "global"])
def test_small_shapes_equal_scipy(harness, shared):
    mats, kinds = _problems(10 + shared, SHAPES, 14)
    assert len(mats) > 2000
    _check(harness, mats, shared, "small", kinds)


@pytest.mark.gpu
def test_512_in_shared_memory_equals_scipy(harness):
    mats, kinds = _problems(20, LARGE, 1)
    _check(harness, mats, 1, "512 shared", kinds)


@pytest.mark.gpu
def test_signed_zero_ties_equal_scipy(harness):
    """Matrices of nothing but -0.0 and +0.0 (and a few -IoU entries), at widths around the warp size."""
    rng = np.random.default_rng(30)
    mats = []
    for nr, nc in [(31, 32), (32, 33), (33, 31), (64, 65), (65, 64), (5, 96), (96, 5)]:
        for _ in range(20):
            c = _signed_zeros(rng, (nr, nc))
            if rng.random() < 0.5:
                k = rng.integers(0, nr * nc, 3)
                c.ravel()[k] = -0.5
            mats.append(c)
    _check(harness, mats, 1, "signed zeros")
    _check(harness, mats, 0, "signed zeros, global")


@pytest.mark.gpu
def test_large_problem_in_global_memory_equals_scipy(harness):
    """IDTP's shape: gt ids x tracker ids of a long sequence, beyond what shared memory holds."""
    rng = np.random.default_rng(40)
    # IDTP's costs are negated counts of frames two ids were matched in: mostly -0.0, a few ids overlapping a lot
    c = -np.where(rng.random((1500, 1400)) < 0.004, rng.integers(1, 60, (1500, 1400)), 0).astype(np.float64)
    d = -rng.integers(0, 6, (1400, 1500)).astype(np.float64)
    _check(harness, [c, d], 0, "large global")
