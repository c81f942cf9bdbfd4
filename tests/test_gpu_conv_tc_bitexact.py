"""The tensor-core conv kernel's outputs, bit for bit, against fixtures recorded from an earlier build
(tests/golden/conv_tc_bitexact.npz, written by tests/golden/make_conv_tc_bitexact.py).

Changes to the mechanics of conv_tc_kernel (loads, splits, barriers, epilogue) must leave every output bit where it was:
the MMAs into each accumulator run in a fixed order, so any difference means the arithmetic changed.  Checked in all three
tensor-core modes on seeded inputs:
  - every tensor-core GEMM of cfg 2 (yolo_mobilev1-0.75, batch 32) one layer at a time through the k2y_conv2d hook;
  - the head tensors of the cfg 2, 3 and 5 networks (yolo_mobilev1-0.75, tiny_yolo, Darknet-53) on seeded batches;
  - the detections `bench.py --dump-outputs` writes for cfg 2 (the last timed step of `--steps 50 --warmup 5 --no-cpu`).
The fixtures hold SHA-256 digests of the output bytes (the full tensors would be tens of megabytes).  They were recorded
from the build of commit 4e4b738, the last one whose consumers issued 64-column plus 16-column wgmmas per tile; the later
whole-width wgmmas are required to reproduce them bit for bit."""
import ctypes
import hashlib
import importlib.util
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from k210_yolo_framework_b200 import _lib, yolonet
from k210_yolo_framework_b200._lib import check, lib
from k210_yolo_framework_b200.weights import random_weights

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "conv_tc_bitexact.npz")
MODES = {"tf32": _lib.MATH_TC_TF32, "3xtf32": _lib.MATH_TC_3XTF32, "bf16x3": _lib.MATH_TC_BF16X3}


def _cfg2_gemms():
    """Every tensor-core GEMM of cfg 2 (M, N, K, ksize): the list the tile-planner tests pin, loaded from that file."""
    spec = importlib.util.spec_from_file_location("_planner_tests", os.path.join(HERE, "test_tile_planner.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.CFG2_GEMMS


CFG2_GEMMS = _cfg2_gemms()
BENCH_ARGS = ["--gpus", "1", "--steps", "50", "--warmup", "5", "--no-cpu"]
BENCH_DUMPS = ("det_index", "det_box_score", "det_counts")
# (cfg, model, alpha, classes, input hw, batch)
NETS = [(2, "yolo_mobilev1", 0.75, 20, (224, 320), 4), (3, "tiny_yolo", 1.0, 20, (416, 416), 2), (5, "yolo", 1.0, 80, (608, 608), 1)]


def digest(t: torch.Tensor) -> np.ndarray:
    return np.frombuffer(hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).digest(), np.uint8)


def gemm_key(mode, M, N, K, ks):
    return f"gemm_{mode}_{M}x{N}x{K}_k{ks}"


def run_gemm(mode, M, N, K, ks):
    """One cfg-2 conv of this GEMM shape through k2y_conv2d: 3x3 layers at batch 32 on their feature map (7x10, 14x20), 1x1
    layers as one row of M pixels; leaky activation, folded BN constants, seeded inputs and weights."""
    if ks == 1:
        B, h, w, cin = 1, 1, M, K
    else:
        h, w = {70: (7, 10), 280: (14, 20)}[M // 32]
        B, cin = 32, K // 9
    rng = np.random.default_rng(M * 7 + N * 3 + K)
    x = torch.from_numpy(rng.standard_normal((B, h, w, cin), dtype=np.float32)).cuda()
    kernel = (rng.standard_normal((ks, ks, cin, N)) / np.sqrt(K)).astype(np.float32)
    scale = (1.0 + 0.1 * rng.standard_normal(N)).astype(np.float32)
    shift = (0.1 * rng.standard_normal(N)).astype(np.float32)
    out = torch.empty(M, N, device="cuda")
    st = torch.cuda.current_stream()
    check(lib.k2y_conv2d(x.data_ptr(), None, None, out.data_ptr(), kernel.ctypes.data, scale.ctypes.data, shift.ctypes.data, B, h, w,
                         cin, 0, 0, N, ks, 1, 0, 1, 0.1, MODES[mode], ctypes.c_void_p(st.cuda_stream)))
    return out


def net_key(mode, cfg, i):
    return f"net_cfg{cfg}_{mode}_head{i}"


def run_net(mode, cfg, model, alpha, classes, hw, batch):
    m, _ = getattr(yolonet, model)([hw[0], hw[1], 3], 3, classes, alpha=alpha, max_batch=batch)
    m.set_weights_dict(random_weights(m.engine.expected_variables(), seed=7, detection_rich=True))
    m.engine.set_math(MODES[mode])
    x = np.random.default_rng(11 + cfg).random((batch, hw[0], hw[1], 3), dtype=np.float32)
    return [torch.as_tensor(h) for h in m.predict_device(torch.from_numpy(x).cuda())]


def bench_dump_digests(out_dir):
    """Runs bench.py (cfg 2, its default bf16x3 mode) with --dump-outputs out_dir; digests of the dumped arrays."""
    r = subprocess.run([sys.executable, os.path.join(os.path.dirname(HERE), "bench.py")] + BENCH_ARGS + ["--dump-outputs", out_dir],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:]
    return {f"bench_{f}": digest(torch.from_numpy(np.load(os.path.join(out_dir, f + ".npy")))) for f in BENCH_DUMPS}


def all_digests(tmp_dir):
    out = {}
    for mode in MODES:
        for g in CFG2_GEMMS:
            out[gemm_key(mode, *g)] = digest(run_gemm(mode, *g))
        for cfg, *net in NETS:
            for i, h in enumerate(run_net(mode, cfg, *net)):
                out[net_key(mode, cfg, i)] = digest(h)
    out.update(bench_dump_digests(tmp_dir))
    return out


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("gemm", CFG2_GEMMS, ids=lambda g: "x".join(map(str, g)))
def test_cfg2_gemm_bit_identical(golden, mode, gemm):
    assert np.array_equal(digest(run_gemm(mode, *gemm)), golden[gemm_key(mode, *gemm)]), f"{mode} {gemm}: output bits changed"


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("net", NETS, ids=lambda n: f"cfg{n[0]}")
def test_head_tensors_bit_identical(golden, mode, net):
    cfg = net[0]
    heads = run_net(mode, *net)
    for i, h in enumerate(heads):
        assert np.array_equal(digest(h), golden[net_key(mode, cfg, i)]), f"cfg {cfg} {mode}: head {i} bits changed"


def test_bench_detections_identical(golden, tmp_path):
    got = bench_dump_digests(str(tmp_path))
    for k, v in got.items():
        assert np.array_equal(v, golden[k]), f"bench --dump-outputs: {k} changed"
