"""CPU tests of face analysis: the ONNX reader / writer (omg_b200/onnx.py) on hand-built and torch-exported graphs, the
executor's load-time checks, the numpy restatement of insightface's contract (oracle/face.py) on hand-built cases,
the product's host steps against it, and the argument checks of the face.cu entry points."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from omg_b200 import _lib as L
from omg_b200 import face as ff
from omg_b200 import onnx as ox
from oracle import face as of
from util_face import export, face_image, tiny_iresnet, tiny_scrfd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _graph_with_shape_chain():
    """x -> Conv -> Shape -> Gather(0) / Gather(2,3) -> Unsqueeze -> Concat(-1 ...) -> Reshape: an exporter-style
    shape subgraph, plus attributes of every supported type."""
    g = np.random.default_rng(0)
    w = g.standard_normal((8, 3, 3, 3)).astype(np.float32)
    nodes = [
        ox.Node("Conv", ["x", "w"], ["c"], "conv0", {"kernel_shape": [3, 3], "pads": [1, 1, 1, 1], "strides": [1, 1]}),
        ox.Node("Shape", ["c"], ["s"], "shape0"),
        ox.Node("Constant", [], ["i0"], "k0", {"value": np.array(0, dtype=np.int64)}),
        ox.Node("Gather", ["s", "i0"], ["b"], "g0", {"axis": 0}),
        ox.Node("Unsqueeze", ["b"], ["b1"], "u0", {"axes": [0]}),
        ox.Node("Constant", [], ["m1"], "k1", {"value": np.array([-1], dtype=np.int64)}),
        ox.Node("Concat", ["b1", "m1"], ["shp"], "cat0", {"axis": 0}),
        ox.Node("Reshape", ["c", "shp"], ["y"], "r0"),
        ox.Node("Identity", ["y"], ["z"], "id0", {"alpha": 0.5, "names": "abc", "fl": [1.0, 2.5]}),
    ]
    gr = ox.Graph(nodes, {"w": w}, [ox.ValueInfo("x", 1, [1, 3, "h", "w"])], [ox.ValueInfo("z", 1, ["n", "m"])], "t")
    return ox.Model(gr, opset=11, ir_version=6, producer="test")


def test_writer_reader_round_trip_is_lossless():
    m = _graph_with_shape_chain()
    m2 = ox.loads(ox.dumps(m))
    assert ox.dumps(m2) == ox.dumps(m)
    assert m2.opset == 11 and m2.graph.inputs[0].shape == [1, 3, "h", "w"]
    np.testing.assert_array_equal(m2.graph.initializers["w"], m.graph.initializers["w"])
    a = m2.graph.nodes[-1].attrs
    assert a["alpha"] == 0.5 and a["names"] == b"abc" and a["fl"] == [1.0, 2.5]
    assert m2.graph.nodes[2].attrs["value"].dtype == np.int64


def test_reader_decodes_float_and_int64_data_fields():
    t = ox._wpacked_ints(1, [2, 2]) + ox._wint(2, 1) + ox._wstr(8, "f") + ox._wbytes(4, np.arange(4, dtype="<f4").tobytes())
    name, arr = ox.parse_tensor(t)
    np.testing.assert_array_equal(arr, np.arange(4, dtype=np.float32).reshape(2, 2))
    t = ox._wpacked_ints(1, [3]) + ox._wint(2, 7) + ox._wstr(8, "i") + ox._wpacked_ints(7, [5, -1, 1 << 40])
    np.testing.assert_array_equal(ox.parse_tensor(t)[1], np.array([5, -1, 1 << 40]))


def test_reader_rejects_external_data_and_unknown_types():
    ext = ox._wpacked_ints(1, [2]) + ox._wint(2, 1) + ox._wstr(8, "big") + ox._wbytes(13, b"")
    with pytest.raises(ValueError, match="'big'.*external_data"):
        ox.parse_tensor(ext)
    bad = ox._wpacked_ints(1, [2]) + ox._wint(2, 16) + ox._wstr(8, "bf") + ox._wbytes(9, b"\0" * 4)
    with pytest.raises(ValueError, match="'bf'.*data_type 16"):
        ox.parse_tensor(bad)


def test_host_shape_subgraph_evaluates_to_torch_shapes():
    m = _graph_with_shape_chain()
    net = ff.OnnxNet(m, device="cpu")
    shape_c = np.array([2, 8, 5, 7], dtype=np.int64)   # what the conv output would be for a (2, 3, 5, 7) input
    env = {"s": shape_c}
    for n in m.graph.nodes[2:7]:
        ins = [env.get(x, net.init.get(x)) for x in n.inputs]
        env[n.outputs[0]] = net._host(n, ins) if n.op_type != "Constant" else net.init[n.outputs[0]]
    assert env["shp"].tolist() == list(torch.zeros(2, 8, 5, 7).reshape(2, -1).shape[:1]) + [-1]


@pytest.mark.parametrize("which", ["iresnet", "scrfd"])
def test_torch_exported_graphs_load_with_every_node_recognised(which):
    if which == "iresnet":
        b = export(tiny_iresnet(0), torch.randn(1, 3, 112, 112))
    else:
        b = export(tiny_scrfd(0), torch.randn(1, 3, 64, 64), dynamic_hw=True)
    m = ox.loads(b)
    net = ff.OnnxNet(m, device="cpu")
    ops = {n.op_type for n in m.graph.nodes}
    assert "BatchNormalization" in ops and "Conv" in ops
    folded = {m.graph.nodes[i].op_type for i in net.skip}
    assert "BatchNormalization" in folded
    if which == "iresnet":
        assert "Flatten" in folded   # Flatten -> Gemm: permuted FC weight
        assert any(m.graph.nodes[i].op_type == "BatchNormalization" for i in net.plan)   # bn1 in front of a padded conv
        assert ff.input_norm_of(m) == (127.5, 127.5)
    else:
        assert {"Resize", "AveragePool", "MaxPool", "Sigmoid"} <= ops
        assert len(m.graph.outputs) == 9


def _one_node_model(node, inits):
    g = ox.Graph([node], inits, [ox.ValueInfo("x", 1, [1, 8, 8, 8])], [ox.ValueInfo("y", 1, None)])
    return ox.Model(g)


def test_executor_rejects_unsupported_ops_and_conv_forms():
    w = np.zeros((8, 8, 3, 3), dtype=np.float32)
    with pytest.raises(NotImplementedError, match="'lrn0'.*LRN"):
        ff.OnnxNet(_one_node_model(ox.Node("LRN", ["x"], ["y"], "lrn0", {"size": 3}), {}), device="cpu")
    with pytest.raises(NotImplementedError, match="'c1'.*asymmetric pads"):
        ff.OnnxNet(_one_node_model(ox.Node("Conv", ["x", "w"], ["y"], "c1", {"pads": [0, 0, 1, 1]}), {"w": w}), device="cpu")
    with pytest.raises(NotImplementedError, match="'c2'.*groups"):
        ff.OnnxNet(_one_node_model(ox.Node("Conv", ["x", "w"], ["y"], "c2", {"group": 2}), {"w": w}), device="cpu")
    w5 = np.zeros((8, 8, 5, 5), dtype=np.float32)
    with pytest.raises(NotImplementedError, match="'c3'.*kernel"):
        ff.OnnxNet(_one_node_model(ox.Node("Conv", ["x", "w"], ["y"], "c3", {}), {"w": w5}), device="cpu")


def test_umeyama_recovers_a_similarity_and_equals_least_squares():
    g = np.random.default_rng(1)
    src = g.uniform(0, 100, (5, 2))
    ang, s, t = 0.3, 1.7, np.array([4.0, -9.0])
    R = np.array([[np.cos(ang), -np.sin(ang)], [np.sin(ang), np.cos(ang)]])
    dst = s * src @ R.T + t
    for fn in (of.umeyama, ff.umeyama):
        T = fn(src, dst)
        np.testing.assert_allclose(T[:2, :2], s * R, atol=1e-9)
        np.testing.assert_allclose(T[:2, 2], t, atol=1e-9)
    noisy = dst + g.normal(0, 2.0, dst.shape)
    # x' = a x - b y + tx, y' = b x + a y + ty in least squares
    A = np.zeros((10, 4))
    A[0::2] = np.c_[src[:, 0], -src[:, 1], np.ones(5), np.zeros(5)]
    A[1::2] = np.c_[src[:, 1], src[:, 0], np.zeros(5), np.ones(5)]
    a, b, tx, ty = np.linalg.lstsq(A, noisy.reshape(-1), rcond=None)[0]
    for fn in (of.umeyama, ff.umeyama):
        np.testing.assert_allclose(fn(src, noisy)[:2], [[a, -b, tx], [b, a, ty]], atol=1e-9)


def test_norm_crop_equals_warp_affine():
    import cv2
    img = face_image(300, 280, 3)
    kps = of.ARCFACE_DST * 1.8 + np.array([20.0, 15.0], dtype=np.float32)
    M = of.umeyama(kps, of.ARCFACE_DST)[:2]
    ref = cv2.warpAffine(img, M, (112, 112), borderValue=0.0)
    np.testing.assert_array_equal(of.norm_crop(img, kps), ref)
    np.testing.assert_array_equal(ff.norm_crop(img, kps), ref)


@pytest.mark.parametrize("hw,scale", [((800, 600), 640 / 800), ((600, 800), 480 / 600), ((500, 500), 640 / 500),
                                      ((1024, 1024), 0.625)])
def test_detection_preprocessing(hw, scale):
    img = face_image(*hw, seed=2)
    c1, s1 = of.det_preprocess(img)
    c2, s2 = ff.det_preprocess(img, (640, 640))
    assert c1.shape == (640, 640, 3) and s1 == pytest.approx(scale) and s1 == s2
    np.testing.assert_array_equal(c1, c2)
    nh, nw = int(round(hw[0] * s1)), int(round(hw[1] * s1))
    assert not c1[nh + 1:].any() and not c1[:, nw + 1:].any()


def _heads(boxes, scores, stride=8, fh=2, fw=2, A=1):
    """Raw heads of one level with hand-set anchors: boxes as distances (l, t, r, b) in strides."""
    n = fh * fw * A
    s = np.zeros((n, 1), np.float32)
    b = np.ones((n, 4), np.float32)
    for i, (sc, bx) in enumerate(zip(scores, boxes)):
        s[i], b[i] = sc, bx
    return [s, b, np.zeros((n, 10), np.float32)]


def _detect(scores, boxes, thresh=0.5):
    s, b, k = _heads(boxes, scores)
    return of.detect_from_outputs([s, b, k], 16, 16, 1.0, thresh, strides=(8,), num_anchors=1)


@pytest.mark.parametrize("x,kept", [(4.25, 1), (4.32, 2), (4.1, 1)])
def test_nms_plus_one_convention_around_0_4(x, kept):
    # A = [0, 0, 9, 9] (area 100 with the +1 convention), B = A shifted by x: IoU = 10 (10 - x) / (200 - 10 (10 - x)):
    # 0.4035 at x = 4.25 (suppressed), 0.3966 at 4.32 (kept).  At x = 4.1 the +1 IoU is 0.418 while the plain one
    # (widths 9) is 0.374: only the +1 convention suppresses B.
    dets = np.array([[0, 0, 9, 9, 0.9], [x, 0, x + 9, 9, 0.8]], dtype=np.float32)
    assert len(of.nms(dets, 0.4)) == kept


def test_score_exactly_at_threshold_is_kept_and_empty_result():
    det, kps = _detect([0.5, 0.49999997], [[1, 1, 1, 1], [1, 1, 1, 1]])
    assert det.shape[0] == 1 and det[0, 4] == np.float32(0.5)
    det, kps = _detect([0.1, 0.2], [[1, 1, 1, 1], [1, 1, 1, 1]])
    assert det.shape == (0, 5) and kps.shape == (0, 5, 2)


def test_all_anchors_above_threshold():
    s = [0.9, 0.8, 0.7, 0.6]
    det, _ = _detect(s, [[0.1, 0.1, 0.1, 0.1]] * 4)   # tiny boxes: nothing overlaps, everything is kept in score order
    assert det[:, 4].tolist() == pytest.approx(s)


def test_face_c_abi_rejects_bad_arguments_before_touching_the_gpu():
    lib = L.load()
    f = C.c_void_p(0x1000)

    def err(rc):
        assert rc == 1
        return lib.omg_last_error().decode()

    assert "unknown activation 7" in err(lib.omg_channel_op(f, 8, f, 8, None, None, None, None, 0, 0, 1, 2, 2, 8, 7, 0, None))
    assert "PReLU needs a slope" in err(lib.omg_channel_op(f, 8, f, 8, None, None, None, None, 0, 0, 1, 2, 2, 8, 2, 0, None))
    assert "even H and W" in err(lib.omg_channel_op(f, 8, f, 8, None, None, None, f, 8, 2, 1, 3, 2, 8, 0, 0, None))
    assert "row strides" in err(lib.omg_channel_op(f, 4, f, 8, None, None, None, None, 0, 0, 1, 2, 2, 8, 0, 0, None))
    assert "multiple of 8" in err(lib.omg_pool2d(f, f, 1, 8, 8, 12, 3, 2, 1, 0, 0, 1, None))
    assert "kernel 5" in err(lib.omg_pool2d(f, f, 1, 8, 8, 16, 5, 2, 1, 0, 0, 1, None))
    d = L.ScrfdDesc()
    d.n_levels, d.num_anchors = 3, 2
    d.out, d.count, d.det_scale, d.nms_thresh = 0x1000, 0x1000, 1.0, 0.4
    for i, s in enumerate((8, 16, 32)):
        d.scores[i] = d.boxes[i] = d.kps[i] = 0x1000
        d.stride[i], d.fh[i], d.fw[i] = s, 704 // s, 704 // s
    d.max_out = 1 << 20
    assert "exceed the 17800" in err(lib.omg_scrfd_detect(C.byref(d), None))
    for i in range(3):
        d.fh[i] = d.fw[i] = 640 // (8 << i)
    d.max_out = 100
    assert "max_out=100 is below the 16800" in err(lib.omg_scrfd_detect(C.byref(d), None))
    d.kps[1] = None
    assert "key-points on some levels" in err(lib.omg_scrfd_detect(C.byref(d), None))
    assert "null descriptor" in err(lib.omg_scrfd_detect(None, None))


def test_pool2d_out_size_equals_torch_output_shape():
    """ops.pool2d_out_size (the host's copy of omg_pool2d's output extent) against torch's max / avg pooling, for every
    window the entry point accepts and inputs of 1 to 12 pixels."""
    from omg_b200 import ops
    n_checked = 0
    for n in range(1, 13):
        for k in (1, 2, 3):
            for stride in (1, 2):
                for pad in (0, 1):
                    if 2 * pad > k or n + 2 * pad < k:
                        continue
                    for ceil in (False, True):
                        x = torch.zeros(1, 1, n, n + 1)
                        want = torch.nn.functional.max_pool2d(x, k, stride, pad, ceil_mode=ceil).shape[2:]
                        assert want == torch.nn.functional.avg_pool2d(x, k, stride, pad, ceil_mode=ceil).shape[2:]
                        got = (ops.pool2d_out_size(n, k, stride, pad, ceil), ops.pool2d_out_size(n + 1, k, stride, pad, ceil))
                        assert got == tuple(want), (n, k, stride, pad, ceil)
                        n_checked += 1
    assert n_checked == 228


def test_face_cu_compiles_without_spills():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    from omg_b200 import build as b
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([nvcc, *b.NVCC_FLAGS, "-c", os.path.join(b.CSRC, "face.cu"), "-o", os.path.join(d, "f.o")],
                           capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(spills) == 4 and all(a == "0" and b_ == "0" for a, b_ in spills)
