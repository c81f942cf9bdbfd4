"""CUDA network path vs the oracle — through the reference-facing builder API / C-ABI."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from k210_yolo_framework_b200 import _lib, yolonet
from k210_yolo_framework_b200.weights import random_weights
from oracle import decode_ref, keras_ref

MODES = [_lib.MATH_FP32_SIMT, _lib.MATH_TC_3XTF32, _lib.MATH_TC_BF16X3]
# per-layer error budget relative to the layer's max |activation| (fp64 oracle): fp32-class modes vs the ~16-bit-mantissa bf16x3
LAYER_TOL = {_lib.MATH_FP32_SIMT: 2e-4, _lib.MATH_TC_3XTF32: 2e-4, _lib.MATH_TC_BF16X3: 6e-4}


def _maxerr(a, b):
    return float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max())


@pytest.mark.parametrize("math", MODES)
def test_mobilev1_real_weights_layerwise(golden_weights, dog_u8, dog_heads, math):
    """Every conv layer of the trained yolo_mobilev1-0.75 on data/dog.jpg against the fp64 oracle."""
    x = (dog_u8 / np.max(dog_u8)).astype(np.float32)[None]
    m, w = yolonet.yolo_mobilev1([224, 320, 3], 3, 20, alpha=0.75, max_batch=2)
    m.engine.set_keep_all(True)
    m.engine.set_use_graph(False)
    m.set_weights_dict(golden_weights)
    m.engine.set_math(math)
    heads = m.predict(x)
    _, acts = keras_ref.forward("yolo_mobilev1", golden_weights, x.astype(np.float64), alpha=0.75,
                                dtype=torch.float64, record=True)
    worst = {}
    for L in m.engine.layers():
        name, bn = L.name.decode(), L.bn_name.decode()
        got = m.engine.read_layer(name, 1)
        # the engine stores the post-BN/activation tensor; pick the oracle's matching record
        if name.startswith("conv_dw_"):
            key = name + "_relu"
        elif name.startswith("conv_pw_") or name == "conv1":
            key = name + "_relu"
        elif bn:
            key = bn + "/leaky"
        else:
            key = name
        ref = acts[key].permute(0, 2, 3, 1).numpy()
        assert got.shape == ref.shape, name
        scale = max(1.0, float(np.abs(ref).max()))
        err = _maxerr(got, ref) / scale
        worst[name] = err
        assert err < LAYER_TOL[math], f"{name}: rel-to-max error {err:.3e} ({_lib.MATH_NAMES[math]})"
    # heads: absolute logit error well inside the 1e-3 score/box budget
    e0, e1 = _maxerr(heads[0], dog_heads["l0_f64"]), _maxerr(heads[1], dog_heads["l1_f64"])
    print(f"[{_lib.MATH_NAMES[math]}] head logit max abs error vs fp64 oracle: {e0:.2e} {e1:.2e}; worst layer {max(worst.values()):.2e}")
    assert e0 < 1e-3 and e1 < 1e-3
    # wrapper view
    hw = w.predict(x)
    assert hw[0].shape == (1, 7, 10, 3, 25) and hw[1].shape == (1, 14, 20, 3, 25)
    np.testing.assert_array_equal(hw[0].reshape(heads[0].shape), heads[0])


CASES = [("yolo_mobilev1", 0.75, 20, (224, 320), 3), ("yolo_mobilev1", 1.0, 20, (96, 128), 2),
         ("yolo_mobilev2", 1.0, 20, (224, 320), 2), ("yolo_mobilev2", 0.5, 20, (96, 96), 2),
         ("tiny_yolo", 1.0, 20, (160, 160), 2), ("yolo", 1.0, 80, (96, 96), 2),
         ("yolo_mobilev1", 0.5, 20, (96, 160), 2)]   # partial tiles on the 48x80 ... 6x10 maps, C = 16..512


@pytest.mark.parametrize("math", MODES)
@pytest.mark.parametrize("model_def,alpha,classes,hw,batch", CASES)
def test_random_weights_all_models(model_def, alpha, classes, hw, batch, math):
    m, _ = getattr(yolonet, model_def)([hw[0], hw[1], 3], 3, classes, alpha=alpha, max_batch=batch)
    weights = random_weights(m.engine.expected_variables(), seed=7, detection_rich=True)
    m.set_weights_dict(weights)
    m.engine.set_math(math)
    x = np.random.default_rng(11).random((batch, hw[0], hw[1], 3), dtype=np.float32)
    got = m.predict(x)
    ref = keras_ref.forward(model_def, weights, x.astype(np.float64), alpha=alpha, dtype=torch.float64)
    for g, r in zip(got, ref):
        assert g.shape == r.shape
        scale = max(1.0, float(np.abs(r).max()))
        assert _maxerr(g, r) / scale < LAYER_TOL[math], f"{model_def} {_lib.MATH_NAMES[math]}: {_maxerr(g, r):.3e} (max |ref| {scale:.2f})"
    # the contract (north_star): decoded confidences and normalised box coordinates within 1e-3 of the reference's
    L = len(got)
    anchors = np.stack([[[0.76, 0.57], [0.69, 0.89], [0.47, 0.34]]] * L) / np.array([1.0, 2.0, 4.0])[:L, None, None]
    h = decode_ref.HelperRef(anchors, list(hw), [(t.shape[1], t.shape[2]) for t in got], classes)
    for b in range(batch):
        gb, gs = decode_ref.decode_layers([t[b].reshape(t.shape[1], t.shape[2], 3, 5 + classes) for t in got], h, list(hw), hw)
        rb, rs = decode_ref.decode_layers([t[b].astype(np.float32).reshape(t.shape[1], t.shape[2], 3, 5 + classes) for t in ref], h, list(hw), hw)
        assert _maxerr(gs, rs) < 1e-3, f"{model_def} {_lib.MATH_NAMES[math]}: score error {_maxerr(gs, rs):.2e}"
        norm = np.array([hw[0], hw[1], hw[0], hw[1]], np.float64)
        box_err = np.abs(gb / norm - rb / norm) / np.maximum(1.0, np.abs(rb / norm))     # relative for boxes wider than the image
        assert float(box_err.max()) < 1e-3, f"{model_def} {_lib.MATH_NAMES[math]}: normalised box error {float(box_err.max()):.2e}"


def _record_key(model_def, name, bn, acts):
    """The oracle record (keras_ref.forward(..., record=True)) of the tensor the engine stores as layer `name`'s output —
    post-BN/activation, plus the block input where the layer adds one — or None when the family has no such layer."""
    if model_def == "yolo_mobilev1" and (name.startswith(("conv_dw_", "conv_pw_")) or name == "conv1"):
        return name + "_relu"
    if model_def == "yolo_mobilev2":
        if name == "Conv1":
            return "Conv1_relu"
        if name == "Conv_1":
            return "out_relu"
        if name.endswith(("_expand", "_depthwise")):
            return name + "_relu"
        if name.endswith("_project"):   # linear bottleneck: BN, no activation; the residual blocks record the add
            add = name[:-len("project")] + "add"
            return add if add in acts else bn
    if bn.startswith("batch_normalization"):
        return bn + "/leaky"
    if name.startswith("conv2d") and not bn:   # a head's output conv (with bias)
        return name
    return None


def _darknet_residual_layers():
    """Creation-order indices of Darknet-53's residual 3x3 convs (the engine adds the block input in their epilogue; the
    oracle records only the conv branch)."""
    i, out = 1, []
    for blocks in (1, 2, 8, 8, 4):
        i += 1                   # the stride-2 downsample conv
        for _ in range(blocks):
            out.append(i + 1)    # the block's 1x1, then its 3x3
            i += 2
    return out


LAYERWISE = [("yolo_mobilev2", 1.0, 20, (224, 320), 2), ("yolo_mobilev2", 0.5, 20, (96, 96), 2),
             ("tiny_yolo", 1.0, 20, (160, 160), 2), ("yolo", 1.0, 80, (96, 96), 2)]
_LAYERWISE_ORACLE = {}   # (case) -> (weights, input, oracle records) of the case last run; the math mode varies fastest


@pytest.mark.parametrize("math", MODES)
@pytest.mark.parametrize("model_def,alpha,classes,hw,batch", LAYERWISE)
def test_random_weights_layerwise(model_def, alpha, classes, hw, batch, math):
    """Every layer of the other families against the fp64 oracle, so that an error in a depthwise (stride 1 and 2, odd
    maps), max-pool (stride 1 and 2), pixel-pair 1x1, residual or concat/upsample layer shows at that layer."""
    m, _ = getattr(yolonet, model_def)([hw[0], hw[1], 3], 3, classes, alpha=alpha, max_batch=batch)
    m.engine.set_keep_all(True)
    m.engine.set_use_graph(False)
    key = (model_def, alpha, classes, hw, batch)
    if key not in _LAYERWISE_ORACLE:      # the fp64 oracle of a network runs once for its three math modes
        _LAYERWISE_ORACLE.clear()
        weights = random_weights(m.engine.expected_variables(), seed=7, detection_rich=True)
        x = np.random.default_rng(11).random((batch, hw[0], hw[1], 3), dtype=np.float32)
        _, acts = keras_ref.forward(model_def, weights, x.astype(np.float64), alpha=alpha, dtype=torch.float64, record=True)
        _LAYERWISE_ORACLE[key] = weights, x, acts
    weights, x, acts = _LAYERWISE_ORACLE[key]
    m.set_weights_dict(weights)
    m.engine.set_math(math)
    m.predict(x)
    layers = m.engine.layers()
    residual = set(_darknet_residual_layers()) if model_def == "yolo" else set()
    refs = []
    for i, L in enumerate(layers):
        name, bn = L.name.decode(), L.bn_name.decode()
        key = _record_key(model_def, name, bn, acts)
        assert key in acts, f"{model_def}: no oracle record for layer {name} (bn '{bn}')"
        ref = acts[key].permute(0, 2, 3, 1).numpy()
        if i in residual:
            assert L.kh == 3 and layers[i - 1].kh == 1 and L.cout == layers[i - 1].cin, name
            ref = ref + refs[i - 2]      # the input of the block's 1x1
        refs.append(ref)
        got = m.engine.read_layer(name, batch)
        assert got.shape == ref.shape, name
        err = _maxerr(got, ref) / max(1.0, float(np.abs(ref).max()))
        assert err < LAYER_TOL[math], f"{model_def} {name}: rel-to-max error {err:.3e} ({_lib.MATH_NAMES[math]})"
    if model_def == "tiny_yolo":
        # the max-pools (not in layers()): 2x2 'SAME' over the first six convs' outputs, the last with stride 1
        tape = keras_ref._Tape(weights, torch.float64)
        for k, stride in enumerate((2, 2, 2, 2, 2, 1)):
            sfx = f"_{k}" if k else ""
            ref = tape.maxpool_same(acts[f"batch_normalization{sfx}/leaky"], stride).permute(0, 2, 3, 1).numpy()
            got = m.engine.read_layer(f"max_pooling2d{sfx}", batch)
            assert got.shape == ref.shape, f"max_pooling2d{sfx}"
            err = _maxerr(got, ref) / max(1.0, float(np.abs(ref).max()))
            assert err < LAYER_TOL[math], f"max_pooling2d{sfx}: rel-to-max error {err:.3e} ({_lib.MATH_NAMES[math]})"


def test_device_api_graph_replay_and_batching():
    m, _ = yolonet.yolo_mobilev1([224, 320, 3], 3, 20, alpha=0.75, max_batch=4)
    weights = random_weights(m.engine.expected_variables(), seed=5, detection_rich=True)
    m.set_weights_dict(weights)
    x = torch.rand((4, 224, 320, 3), device="cuda")
    a = [t.clone() for t in m.predict_device(x)]          # captures the graph for batch 4
    b = [t.clone() for t in m.predict_device(x)]          # replays it
    for p, q in zip(a, b):
        assert torch.equal(p, q)
    c = [t.clone() for t in m.predict_device(x[1:3])]     # different batch -> second graph; tile / split-K shapes may
    for p, q in zip(a, c):                                 # differ with M, so only the accumulation order changes
        assert torch.allclose(p[1:3], q, atol=2e-4, rtol=1e-4)
    m.engine.set_use_graph(False)
    d = m.predict_device(x)
    for p, q in zip(a, d):
        assert torch.equal(p, q)
    host = m.predict(x.cpu().numpy())
    for p, q in zip(a, host):
        np.testing.assert_array_equal(p.cpu().numpy(), q)
    assert m.engine.launches_per_run() >= 32   # + split-K reducers


def test_predict_after_uint8_input_uses_the_float_input():
    """predict() after a uint8 run must read ITS float32 input, not the uint8 buffer still bound from before."""
    m, _ = yolonet.yolo_mobilev1([224, 320, 3], 3, 20, alpha=0.75, max_batch=2)
    weights = random_weights(m.engine.expected_variables(), seed=5, detection_rich=True)
    m.set_weights_dict(weights)
    rng = np.random.default_rng(0)
    a_u8 = torch.from_numpy(rng.integers(0, 256, (2, 224, 320, 3), dtype=np.uint8)).cuda()
    b = rng.random((2, 224, 320, 3), dtype=np.float32)
    fresh = [t.copy() for t in m.predict(b)]
    m.predict_device_u8(a_u8)
    again = m.predict(b)
    for p, q in zip(fresh, again):
        np.testing.assert_array_equal(p, q)
    # ... and an externally bound input buffer (double-buffered ingest) gives the same heads as the engine's own
    ext = torch.from_numpy(b).cuda()
    m.engine.bind_input(ext)
    via_ext = [t.clone() for t in m.engine.run(2)]
    for p, q in zip(fresh, via_ext):
        np.testing.assert_array_equal(p, q.cpu().numpy())
    m.engine.unbind_input()


def test_errors():
    m, _ = yolonet.yolo_mobilev1([224, 320, 3], 3, 20, alpha=0.75, max_batch=2)
    with pytest.raises(_lib.K2YError):
        m.predict(np.zeros((1, 224, 320, 3), np.float32))            # weights not loaded
    with pytest.raises(ValueError):
        m.set_weights_dict({})
    weights = random_weights(m.engine.expected_variables(), seed=5)
    bad = dict(weights)
    bad["conv1"] = {"kernel": np.zeros((3, 3, 3, 8), np.float32)}
    with pytest.raises(ValueError):
        m.set_weights_dict(bad)
    m.set_weights_dict(weights)
    with pytest.raises(ValueError):
        m.predict(np.zeros((1, 100, 100, 3), np.float32))
    with pytest.raises(ValueError):
        m.predict_device(torch.zeros((3, 224, 320, 3), device="cuda"))  # > max_batch
