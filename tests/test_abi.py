"""The C-ABI library loads without a GPU and exports every symbol the headers declare."""
import ctypes
import os
import re

from conftest import ROOT


def _declared(header):
    src = open(os.path.join(ROOT, "include", header)).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b((?:k2y|region_layer)_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from k210_yolo_framework_b200 import _lib
    lib = ctypes.CDLL(_lib.LIB_PATH)
    names = _declared("k210_yolo_b200.h") + _declared("region_layer.h")
    assert len(names) >= 28
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/ but not exported"


def test_python_binding_covers_header():
    from k210_yolo_framework_b200 import _lib
    assert sorted(_lib._SIGNATURES) == _declared("k210_yolo_b200.h")
    assert sorted(_lib._REGION_ABI) == _declared("region_layer.h")


def test_struct_sizes_match_header():
    from k210_yolo_framework_b200 import _lib
    assert ctypes.sizeof(_lib.Det) == 24
    assert ctypes.sizeof(_lib.LayerInfo) == 64 + 64 + 7 * 4
    assert ctypes.sizeof(_lib.DetectCfg) == 4 + 12 + 12 + 8 + 48 * 4 + 8 + 8 + 4
    assert ctypes.sizeof(_lib.RegionCfg) == 8 * 4 + 16 * 4 + 8


def test_error_reporting_without_gpu():
    from k210_yolo_framework_b200 import _lib
    h = ctypes.c_void_p()
    rc = _lib.lib.k2y_net_create(b"not_a_model", 224, 320, 1.0, 3, 20, 1, 0, ctypes.byref(h))
    assert rc == -1 and "unknown model_def" in _lib.last_error()
    rc = _lib.lib.k2y_net_create(b"yolo_mobilev1", 225, 320, 1.0, 3, 20, 1, 0, ctypes.byref(h))
    assert rc == -1 and "multiple of 32" in _lib.last_error()
    # depthwise widths the float4 kernel cannot run: conv_dw_1 of yolo_mobilev1 gets int(32 * alpha) channels
    for alpha, channels in ((0.35, 11), (0.6, 19)):
        rc = _lib.lib.k2y_net_create(b"yolo_mobilev1", 224, 320, alpha, 3, 20, 1, 0, ctypes.byref(h))
        err = _lib.last_error()
        assert rc == -1 and "conv_dw_1" in err and f"has {channels} channels" in err, err
    rc = _lib.lib.k2y_net_create(b"yolo_mobilev1", 224, 320, 0.25, 3, 20, 1, 0, ctypes.byref(h))   # 8 channels: fine
    assert rc == 0
    _lib.lib.k2y_net_destroy(h)
    assert _lib.lib.k2y_version() >= 100
