#!/usr/bin/env python
"""Per-shape attribution of the tensor-core conv kernel (conv_tc_kernel): every tensor-core GEMM of cfg 2 (yolo_mobilev1-0.75,
320x224, batch 32; CFG2_GEMMS in tests/test_tile_planner.py) through the k2y_conv2d hook on device tensors, in bf16x3.

For each shape it prints the device time of one launch (conv_tc_kernel plus, for split-K plans, the reduce pass), the
tensor-pipe floor of the plan the planner picks (k2y_tc_plan_budget) quantised to the plan's rounds of work items, and the
share of that floor reached.  The card's name, power limit and SM clocks are read in the same run.

Kernel times come from torch.profiler (CUDA activities): k2y_conv2d packs the weights on the host and synchronises around
every launch, so device events around the call would time the host.  Inputs rotate over enough buffers that one layer's
inputs and outputs do not stay in the 50 MB L2 from one launch to the next.

Ablation libraries (built with -DK2Y_TC_ABLATE=N, never the shipped one) attribute the time: 1 = no epilogue stores,
2 = no MMAs (loads, splits and barriers kept), 3 = no A split (raw bits as hi, zero lo), 4 = no B traffic (weight tiles are
loaded for a CTA's first `stages` k-blocks only; the MMAs then read stale ones).

    python scripts/bench_conv_tc.py --build-ablations DIR          # compile the four variants into DIR (no GPU needed)
    python scripts/bench_conv_tc.py [--ablations DIR] [--lib NAME=PATH ...] [--rounds 3] [--launches 200] [--json OUT]

With several libraries the runs alternate (lib a, lib b, ..., lib a, ...) `--rounds` times; each cell is the median.
"""
import argparse
import ctypes
import importlib.util
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MATH_TC_BF16X3, MATH_TC_TF32 = 3, 2
ABLATIONS = {1: "no_epilogue_stores", 2: "no_mma", 3: "no_a_split", 4: "no_b_traffic"}
# tensor-pipe rate per SM and clock (dense, data-sheet): 2048 bf16 MAC, 1024 tf32 MAC
MAC_PER_CLK = {"bf16": 2048, "tf32": 1024}


def cfg2_gemms():
    spec = importlib.util.spec_from_file_location("_planner_tests", os.path.join(ROOT, "tests", "test_tile_planner.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.CFG2_GEMMS


def build_ablations(out_dir):
    spec = importlib.util.spec_from_file_location("_k2y_build", os.path.join(ROOT, "k210_yolo_framework_b200", "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    os.makedirs(out_dir, exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    procs = []
    for n in ABLATIONS:
        out = os.path.join(out_dir, f"libk210yolo_b200_ablate{n}.so")
        cmd = [nvcc] + b.NVCC_FLAGS + [f"-DK2Y_TC_ABLATE={n}", "-o", out] + [os.path.join(b.CSRC, s) for s in b.SOURCES] + ["-ldl"]
        procs.append((out, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for out, p in procs:
        log = p.communicate()[0]
        if p.returncode != 0:
            sys.stderr.write(log)
            raise RuntimeError(f"nvcc failed building {out}")
        print(out)


def load(path):
    lib = ctypes.CDLL(path)
    c_int, c_void_p = ctypes.c_int, ctypes.c_void_p
    lib.k2y_conv2d.restype = c_int
    lib.k2y_conv2d.argtypes = [c_void_p] * 7 + [c_int] * 11 + [ctypes.c_float, c_int, c_void_p]
    lib.k2y_last_error.restype = ctypes.c_char_p
    lib.k2y_tc_plan_budget.restype = c_int
    lib.k2y_tc_plan_budget.argtypes = [c_int] * 6 + [ctypes.POINTER(c_int)] * 6
    return lib


def plan(lib, M, N, K, ks):
    v = [ctypes.c_int() for _ in range(6)]
    if lib.k2y_tc_plan_budget(M, N, K, ks, MATH_TC_BF16X3, 0, *[ctypes.byref(x) for x in v]) != 0:
        raise RuntimeError(lib.k2y_last_error().decode())
    return dict(zip(("bn", "splits", "stages", "cluster", "math", "grid"), (x.value for x in v)))


def floor_us(M, N, K, pl, ghz):
    """Tensor-pipe time of the plan: every work item (128 rows x bn columns x its k-slice) runs at the data-sheet MMA rate,
    and the items run in ceil(items / grid) rounds of one item per CTA.  Zero-padded K and N columns count, as they cost MMAs."""
    bf16 = pl["math"] == MATH_TC_BF16X3
    passes = 1 if pl["math"] == MATH_TC_TF32 else 3
    kbk = 64 if bf16 else 32
    nkb = -(-K // kbk)
    kb_per = -(-nkb // pl["splits"])
    items = -(-M // 128) * -(-(-(-N // 16) * 16) // pl["bn"]) * pl["splits"]
    rounds = -(-items // pl["grid"])
    clk_per_kb = passes * 128 * pl["bn"] * kbk / MAC_PER_CLK["bf16" if bf16 else "tf32"]
    return rounds * kb_per * clk_per_kb / (ghz * 1e3), items, rounds


def geometry(M, K, ks):
    """(batch, h, w, cin) of a cfg-2 conv with this GEMM shape: 3x3 layers at batch 32 on their feature map, 1x1 as one row."""
    if ks == 1:
        return 1, 1, M, K
    hw = M // 32
    h = int(round((hw * 0.7) ** 0.5))
    assert h * (hw // h) == hw, (M, K)
    return 32, h, hw // h, K // 9


class Shape:
    def __init__(self, torch, M, N, K, ks, seed):
        import numpy as np
        self.M, self.N, self.K, self.ks = M, N, K, ks
        self.B, self.h, self.w, self.cin = geometry(M, K, ks)
        rng = np.random.default_rng(seed)
        self.kernel = (rng.standard_normal((ks, ks, self.cin, N)) / (K ** 0.5)).astype(np.float32)
        self.scale = (1.0 + 0.1 * rng.standard_normal(N)).astype(np.float32)
        self.shift = (0.1 * rng.standard_normal(N)).astype(np.float32)
        in_bytes, out_bytes = self.B * self.h * self.w * self.cin * 4, M * N * 4
        nbuf = max(1, -(-(100 << 20) // (in_bytes + out_bytes)))   # >= 100 MB, twice the L2, over the rotation
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.src = [torch.randn(self.B, self.h, self.w, self.cin, device="cuda", generator=g) for _ in range(nbuf)]
        self.dst = [torch.empty(M, N, device="cuda") for _ in range(nbuf)]

    def launch(self, lib, i, stream):
        s, d = self.src[i % len(self.src)], self.dst[i % len(self.dst)]
        rc = lib.k2y_conv2d(s.data_ptr(), None, None, d.data_ptr(), self.kernel.ctypes.data, self.scale.ctypes.data,
                            self.shift.ctypes.data, self.B, self.h, self.w, self.cin, 0, 0, self.N, self.ks, 1, 0, 1, 0.1,
                            MATH_TC_BF16X3, ctypes.c_void_p(stream))
        if rc != 0:
            raise RuntimeError(lib.k2y_last_error().decode())


def time_shape(torch, lib, shape, launches, warmup):
    from torch.profiler import ProfilerActivity, profile
    stream = torch.cuda.current_stream().cuda_stream
    for i in range(warmup):
        shape.launch(lib, i, stream)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(launches):
            shape.launch(lib, i, stream)
        torch.cuda.synchronize()
    # per kernel: (summed us, count); the trace can miss a record at the edge of its window, so each kernel is averaged
    # over the launches it recorded
    seen = {"conv_tc_kernel": [0.0, 0], "splitk_reduce_kernel": [0.0, 0]}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        for k, v in seen.items():
            if k in e.name:
                v[0] += e.time_range.elapsed_us()
                v[1] += 1
    if seen["conv_tc_kernel"][1] < launches - 2:
        raise RuntimeError(f"the profiler saw {seen['conv_tc_kernel'][1]} conv_tc_kernel launches of {launches}")
    return sum(t / n for t, n in seen.values() if n)


def card_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--build-ablations", metavar="DIR", default=None)
    ap.add_argument("--ablations", metavar="DIR", default=None, help="time the variants built by --build-ablations DIR too")
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=PATH", help="a library to time (default: the package's)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--clock-ghz", type=float, default=1.98, help="SM clock of the floor (default: the H100 SXM's maximum)")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if args.build_ablations:
        build_ablations(args.build_ablations)
        return

    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_conv_tc.py needs a CUDA device")
    torch.cuda.set_device(0)
    libs = [tuple(x.split("=", 1)) for x in args.lib] or [("shipped", os.path.join(ROOT, "k210_yolo_framework_b200", "libk210yolo_b200.so"))]
    if args.ablations:
        libs += [(name, os.path.join(args.ablations, f"libk210yolo_b200_ablate{n}.so")) for n, name in ABLATIONS.items()]
    loaded = [(name, load(path)) for name, path in libs]
    card = card_info()

    shapes = [Shape(torch, M, N, K, ks, seed=i) for i, (M, N, K, ks) in enumerate(cfg2_gemms())]
    times = {name: [[] for _ in shapes] for name, _ in loaded}
    for _ in range(args.rounds):
        for si, sh in enumerate(shapes):
            for name, lib in loaded:
                times[name][si].append(time_shape(torch, lib, sh, args.launches, args.warmup))

    ref_lib = loaded[0][1]
    rows = []
    print(f"card: {card}  (floor at {args.clock_ghz} GHz, {MAC_PER_CLK['bf16']} bf16 MAC/clk/SM, 3 MMAs per useful MAC)")
    hdr = f"{'M':>7} {'N':>4} {'K':>5} k  bn sp grid items rnd floor_us " + " ".join(f"{n[:14]:>14}" for n, _ in loaded)
    print(hdr)
    for si, sh in enumerate(shapes):
        pl = plan(ref_lib, sh.M, sh.N, sh.K, sh.ks)
        fl, items, rounds = floor_us(sh.M, sh.N, sh.K, pl, args.clock_ghz)
        med = {name: float(np.median(times[name][si])) for name, _ in loaded}
        cells = " ".join(f"{med[n]:7.2f} ({fl / med[n]:4.0%})" for n, _ in loaded)
        print(f"{sh.M:7d} {sh.N:4d} {sh.K:5d} {sh.ks}  {pl['bn']:3d} {pl['splits']:2d} {pl['grid']:4d} {items:5d} {rounds:3d} {fl:8.2f} {cells}")
        rows.append({"M": sh.M, "N": sh.N, "K": sh.K, "ksize": sh.ks, "plan": pl, "items": items, "rounds": rounds, "floor_us": fl,
                     "us": med, "us_all": {n: times[n][si] for n, _ in loaded}, "share": {n: fl / med[n] for n in med}})
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump({"card": card, "clock_ghz": args.clock_ghz, "launches": args.launches, "rounds": args.rounds,
                       "libs": [n for n, _ in loaded], "shapes": rows}, f, indent=1)


if __name__ == "__main__":
    main()
