"""GPU tests of face analysis on the kernels (omg_b200/face.py, csrc/face.cu): omg_channel_op / omg_pool2d against
torch in fp32, omg_scrfd_detect against the numpy restatement of SCRFD.detect (exactly), the ONNX executor against the
fp32 oracle modules exported by torch (full-depth IResNet-100, the SCRFD-style detector), FaceAnalysis.get against the
oracle's get(), and the InstantID CLI with face analysis from generated model files."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from omg_b200 import _lib as L
from omg_b200 import face as ff
from omg_b200 import ops
from oracle import face as of
from util_face import export, face_image, tiny_iresnet, tiny_scrfd, write_antelopev2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _h(t):
    return t.half().cuda()


@pytest.mark.parametrize("act", [L.CH_ACT_NONE, L.CH_ACT_RELU, L.CH_ACT_PRELU, L.CH_ACT_SIGMOID])
@pytest.mark.parametrize("add_scale", [0, 1, 2])
@pytest.mark.parametrize("after", [False, True])
@pytest.mark.parametrize("C", [24, 5])
def test_channel_op_matches_torch(act, add_scale, after, C):
    g = torch.Generator().manual_seed(C + 10 * add_scale + act)
    B, H, W, ld = 2, 6, 10, (40 if C % 8 == 0 else C)
    xs = torch.randn(B, H, W, ld, generator=g)
    x = _h(xs)[..., :C]
    s, t, sl = (torch.randn(C, generator=g).cuda() for _ in range(3))
    add = None
    if add_scale:
        add = _h(torch.randn(B, H // add_scale, W // add_scale, C, generator=g))
    # output rows of ld channels, poisoned: channels past C must stay untouched
    out = torch.full((B, H, W, ld), 7.0, dtype=torch.float16, device="cuda")
    ops.channel_op(x, scale=s, shift=t, act=act, slope=sl, addend=add, add_scale=max(add_scale, 1), act_after_add=after,
                   out=out[..., :C])
    v = x.float() * s + t
    a = 0 if add is None else add.float().repeat_interleave(add_scale, 1).repeat_interleave(add_scale, 2)
    f = {L.CH_ACT_NONE: lambda z: z, L.CH_ACT_RELU: torch.relu, L.CH_ACT_SIGMOID: torch.sigmoid,
         L.CH_ACT_PRELU: lambda z: torch.where(z >= 0, z, z * sl)}[act]
    ref = f(v + a) if after else f(v) + a
    assert (out[..., :C].float() - ref).abs().max().item() < 2e-2
    assert bool((out[..., C:] == 7.0).all())


@pytest.mark.parametrize("is_max", [True, False])
@pytest.mark.parametrize("k,stride,pad", [(3, 2, 1), (3, 1, 1), (2, 2, 0), (3, 2, 0), (1, 2, 0)])
@pytest.mark.parametrize("ceil_mode", [False, True])
@pytest.mark.parametrize("cip", [False, True])
@pytest.mark.parametrize("hw", [(9, 13), (8, 8)])
def test_pool2d_matches_torch(is_max, k, stride, pad, ceil_mode, cip, hw):
    if is_max and cip:
        pytest.skip("count_include_pad is an average-pool option")
    g = torch.Generator().manual_seed(k * 7 + stride + pad)
    x = torch.randn(2, 16, *hw, generator=g)
    if is_max:
        ref = torch.nn.functional.max_pool2d(x, k, stride, pad, ceil_mode=ceil_mode)
    else:
        ref = torch.nn.functional.avg_pool2d(x, k, stride, pad, ceil_mode=ceil_mode, count_include_pad=cip)
    y = ops.pool2d(_h(x.permute(0, 2, 3, 1).contiguous()), k, stride, pad, ceil_mode, cip, is_max)
    assert y.shape[1:3] == ref.shape[2:]
    assert (y.float().permute(0, 3, 1, 2).cpu() - ref).abs().max().item() < 1e-2


def _raw_heads(seed, fh_fw, A=2, score_mode="rand", thresh=0.5):
    g = np.random.default_rng(seed)
    outs = {"s": [], "b": [], "k": []}
    for fh, fw in fh_fw:
        n = fh * fw * A
        sc = g.random((n, 1)).astype(np.float32) if score_mode == "rand" else \
            (thresh + g.random((n, 1)) * 0.5).astype(np.float32)
        outs["s"].append(sc)
        outs["b"].append((g.random((n, 4)) * 3 + 0.2).astype(np.float32))
        outs["k"].append((g.normal(size=(n, 10)) * 2).astype(np.float32))
    return outs["s"] + outs["b"] + outs["k"]


@pytest.mark.parametrize("case", ["random_64", "all_16800", "ties_and_threshold", "none"])
def test_scrfd_detect_matches_numpy_exactly(case):
    strides = (8, 16, 32)
    size = 640 if case == "all_16800" else 64
    grids = [(size // s, size // s) for s in strides]
    outs = _raw_heads(3, grids, score_mode="all" if case == "all_16800" else "rand")
    if case == "ties_and_threshold":
        outs[0][:40] = 0.5            # exactly at det_thresh, equal scores
        outs[1][:4] = 0.75
    if case == "none":
        outs = [o * (0.3 if i < 3 else 1) for i, o in enumerate(outs)]
    det_scale = 0.4 if size == 640 else 0.8125
    det, kpss = of.detect_from_outputs(outs, size, size, det_scale, 0.5)
    levels = [(s, fh, fw, torch.from_numpy(outs[i]).cuda(), torch.from_numpy(outs[i + 3]).cuda(),
               torch.from_numpy(outs[i + 6]).cuda()) for i, (s, (fh, fw)) in enumerate(zip(strides, grids))]
    rows = ops.scrfd_detect(levels, 2, 0.5, det_scale).cpu().numpy()
    if case == "all_16800":
        assert sum(fh * fw * 2 for fh, fw in grids) == 16800
    assert rows.shape[0] == det.shape[0]
    if case == "none":
        assert rows.shape[0] == 0
    else:
        assert rows.shape[0] > 0
    np.testing.assert_array_equal(rows[:, :5], det)
    np.testing.assert_array_equal(rows[:, 5:], kpss.reshape(-1, 10))


def _rel(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def _cos(a, b):
    return float((a * b).sum() / np.linalg.norm(a) / np.linalg.norm(b))


# measured on an H100 80GB HBM3 (700 W power limit): IResNet-100 rel L2 1.603e-3, cosine 0.999999 (printed to six
# places, so 1 - cos <= 1.5e-6); SCRFD-style detector, worst of the nine outputs 7.06e-4.  Tolerances: these x 1.25.
IRESNET100_REL, IRESNET100_COS = 1.61e-3, 1 - 1.5e-6
SCRFD_OUT_REL = 7.1e-4


def test_iresnet100_onnx_matches_fp32_oracle(tmp_path):
    net = of.randomize_(of.IResNet(), 11)
    x = torch.from_numpy(of.rec_blob([face_image(112, 112, s) for s in range(2)]))
    onnx_bytes = export(net, x[:1])
    rec = ff.ArcFace(model=ff.ox.loads(onnx_bytes))
    with torch.no_grad():
        ref = net(x).numpy()
    got = rec.net.run(ff.image_to_act(x.numpy(), rec.device))[0].cpu().numpy()
    rel, cos = max(_rel(got[i], ref[i]) for i in range(2)), min(_cos(got[i], ref[i]) for i in range(2))
    print(f"IResNet-100 on the kernels vs fp32: rel L2 {rel:.3e}, cosine {cos:.6f}")
    assert rel < IRESNET100_REL * 1.25
    assert cos > 1 - (1 - IRESNET100_COS) * 1.25


def test_scrfd_onnx_matches_fp32_oracle():
    net = of.randomize_(of.ScrfdNet(), 5)
    det_img, _ = of.det_preprocess(face_image(480, 640, 1))
    x = torch.from_numpy(of.det_blob(det_img))
    det = ff.SCRFD(model=ff.ox.loads(export(net, x, dynamic_hw=True)))
    with torch.no_grad():
        ref = [o.numpy() for o in net(x)]
    got = det.forward_raw(det_img)
    errs = [_rel(g.cpu().numpy(), r) for g, r in zip(got, ref)]
    print("SCRFD outputs on the kernels vs fp32: rel L2 " + " ".join(f"{e:.3e}" for e in errs))
    assert all(g.shape == r.shape for g, r in zip(got, ref))
    assert max(errs) < SCRFD_OUT_REL * 1.25


def _margins(outs, det_thresh, det_size, det_scale):
    """Smallest distance of any anchor score to det_thresh, and of any pairwise IoU among the candidates to 0.4."""
    s = np.concatenate([o.reshape(-1) for o in outs[:3]])
    dm = float(np.abs(s - det_thresh).min())
    sc, bx, _ = of.decode(outs, det_size, det_size, det_thresh)
    b = np.concatenate(bx) / np.float32(det_scale)
    area = (b[:, 2] - b[:, 0] + 1) * (b[:, 3] - b[:, 1] + 1)
    iw = np.maximum(0, np.minimum(b[:, None, 2], b[None, :, 2]) - np.maximum(b[:, None, 0], b[None, :, 0]) + 1)
    ih = np.maximum(0, np.minimum(b[:, None, 3], b[None, :, 3]) - np.maximum(b[:, None, 1], b[None, :, 1]) + 1)
    inter = iw * ih
    iou = inter / (area[:, None] + area[None, :] - inter)
    iu = iou[np.triu_indices(len(b), 1)]
    return dm, float(np.abs(iu - 0.4).min()) if iu.size else 1.0, len(b)


def _clear_threshold(outs, delta, max_faces=30):
    """A det_thresh in the widest gap of the top scores (at least 2 delta wide), or None."""
    s = np.sort(np.concatenate([o.reshape(-1) for o in outs[:3]]))[::-1]
    gaps = s[:max_faces] - s[1:max_faces + 1]
    k = int(np.argmax(gaps))
    return float((s[k] + s[k + 1]) / 2) if gaps[k] >= 2 * delta else None


def test_get_matches_oracle_get(tmp_path):
    # an image and a det_thresh where every anchor's score is clear of the threshold and every candidate pair's IoU
    # clear of 0.4 by more than the fp16 network's error, so the comparison cannot hinge on rounding
    d_score, d_iou = 5e-3, 1e-2
    det_net = tiny_scrfd(3, score_bias=-1.45)
    found = None
    for seed in range(12):
        img = face_image(600, 800, seed)
        det_img, det_scale = of.det_preprocess(img)
        with torch.no_grad():
            outs = [o.numpy() for o in det_net(torch.from_numpy(of.det_blob(det_img)))]
        thr = _clear_threshold(outs, d_score)
        if thr is None:
            continue
        dm, im, n = _margins(outs, thr, 640, det_scale)
        if dm >= d_score and im >= d_iou and n >= 1:
            found = (thr, dm, im, n)
            break
    assert found, "no image with every score and IoU clear of the thresholds"
    thr, dm, im, n = found
    print(f"image {seed}, det_thresh {thr:.4f}: {n} candidates, score margin {dm:.2e}, IoU margin {im:.2e}")
    rec_net = tiny_iresnet(4)
    root = write_antelopev2(str(tmp_path), det_net, rec_net)
    app = ff.FaceAnalysis(root=root)
    app.prepare(ctx_id=0, det_thresh=thr, det_size=(640, 640))
    ref = of.get(img, det_net, rec_net, det_thresh=thr)
    got = app.get(img)
    assert len(got) == len(ref) >= 1
    worst = 1.0
    for f, r in zip(got, ref):
        np.testing.assert_allclose(f.bbox, r["bbox"], atol=2.0)
        np.testing.assert_allclose(f.kps, r["kps"], atol=2.0)
        assert abs(float(f.det_score) - float(r["det_score"])) < 2e-2
        # the recogniser on the crop of the detected key-points, against fp32 on the same crop
        with torch.no_grad():
            e32 = rec_net(torch.from_numpy(of.rec_blob([of.norm_crop(img, f.kps)])))[0].numpy()
        assert _cos(f.embedding, e32) > 0.999
        worst = min(worst, _cos(f.embedding, r["embedding"]))
        assert f.normed_embedding.shape == (512,) and abs(np.linalg.norm(f.normed_embedding) - 1) < 1e-5
    print(f"{len(got)} faces; embedding cosine vs the oracle's own crops >= {worst:.5f}")


def test_cli_detects_stage2_keypoints_on_the_stage1_image(tmp_path):
    import cv2
    from PIL import Image
    root = write_antelopev2(str(tmp_path / "antelopev2"), tiny_scrfd(1, score_bias=4.0, box_bias=12.0), tiny_iresnet(2))
    refs = []
    for k in range(2):
        p = str(tmp_path / f"ref{k}.png")
        cv2.imwrite(p, face_image(300, 260, 50 + k))
        refs.append(p)
    rewrite = "|".join(f"[a person]-*-[bad]-*-{p}" for p in refs)
    out = tmp_path / "out"
    cmd = [sys.executable, os.path.join(ROOT, "inference_instantid.py"), "--synthetic", "--tiny", "--decode",
           "--image_size", "256", "--num_inference_steps", "2", "--antelopev2_path", root, "--save_dir", str(out),
           "--prompt_rewrite", rewrite, "--prompt", "two people"]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert "face analysis on the kernels" in r.stdout
    d = out / "seed_53"
    kps = json.load(open(d / "face_kps.json"))
    assert f"stage-1 image: {len(kps)} faces" in r.stdout and len(kps) >= 1
    app = ff.FaceAnalysis(root=root)
    app.prepare(ctx_id=0, det_size=(640, 640))
    stage1 = np.array(Image.open(d / "stage-1.png").convert("RGB"))
    again = app.get(cv2.cvtColor(stage1, cv2.COLOR_RGB2BGR))
    assert len(again) == len(kps)
    np.testing.assert_allclose(np.array([f.kps for f in again]), np.array(kps), atol=1e-4)
    sys.path.insert(0, ROOT)
    from inference_instantid import draw_kps_multi
    cond = np.array(Image.open(d / "stage-2-condition.png"))
    np.testing.assert_array_equal(cond, draw_kps_multi((256, 256), kps))
    assert (d / "stage-2.png").exists()
