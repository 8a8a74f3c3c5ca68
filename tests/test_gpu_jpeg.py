"""GPU: frame decode on the device (csrc/jpeg.cu through nvJPEG) against cv2 (what the reference's loader uses,
lib/utils/image.py:51-63), and the device-fill path of the clip pipeline against the pinned-staging path.
JPEG decoders are not bit-identical (IDCT rounding, chroma upsampling filter): 4:4:4 streams must agree to a few grey levels,
4:2:0 streams on average."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _image(h, w, seed):
    rng = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    im = np.stack([128 + 100 * np.sin(xx / 37.0 + seed), 128 + 100 * np.cos(yy / 23.0), 64 + 0.2 * xx + 0.1 * yy], 2)
    im += rng.normal(0, 6, im.shape)
    return np.clip(im, 0, 255).astype(np.uint8)


def test_jpeg_decode_vs_cv2():
    import cv2
    import torch
    from detectandtrack_b200.ops import image_ops
    if not image_ops.jpeg_available():
        pytest.skip('nvJPEG is not installed on this machine')
    H, W = 240, 328
    ims = [_image(H, W, s) for s in range(3)]
    for tag, flags, mean_tol, max_tol in (('444', [cv2.IMWRITE_JPEG_QUALITY, 92, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444], 0.8, 8),        # nvJPEG vs cv2 rounding
                                           ('420', [cv2.IMWRITE_JPEG_QUALITY, 92], 1.5, 24)):
        streams = [cv2.imencode('.jpg', im, flags)[1].tobytes() for im in ims]
        ref = np.stack([cv2.imdecode(np.frombuffer(s, np.uint8), cv2.IMREAD_COLOR) for s in streams])
        got = image_ops.jpeg_decode(streams, H, W)
        torch.cuda.synchronize()
        d = np.abs(got.cpu().numpy().astype(np.int32) - ref.astype(np.int32))
        print('jpeg %s: mean |diff| %.3f, max %d grey levels vs cv2' % (tag, d.mean(), d.max()))
        assert got.shape == (3, H, W, 3) and d.mean() <= mean_tol and d.max() <= max_tol, (tag, d.mean(), d.max())
    with pytest.raises(RuntimeError, match='expected'):
        image_ops.jpeg_decode(streams, H + 8, W)
    with pytest.raises(RuntimeError, match='not a JPEG'):
        image_ops.jpeg_decode([b'not a jpeg at all' * 10], H, W)


def test_pipeline_device_fill_equals_pinned_staging():
    """The device-fill path of ClipPipeline.run (what TEST.DEVICE_JPEG_DECODE uses) with a plain device copy as the producer:
    same detections as the pinned-staging path, bit for bit, over several steps and a short last batch."""
    import torch
    from test_gpu_engine import _cfg
    from detectandtrack_b200.modeling import model_builder
    from detectandtrack_b200.core.test import get_pipeline
    cfg = _cfg()
    try:
        model = model_builder.create(cfg.MODEL.TYPE, train=False, dtype='bf16x3')
        rng = np.random.RandomState(0)
        clips = rng.randint(0, 256, (7, 3, 96, 128, 3)).astype(np.uint8)
        dev = torch.from_numpy(clips).cuda()
        pipe = get_pipeline(model, 2, 3, 96, 128)
        a, b = [None] * 7, [None] * 7
        pipe.run(7, lambda i, dst: np.copyto(dst, clips[i]), lambda i, *r: a.__setitem__(i, r))

        def fill_device(i, dst, stream):
            with torch.cuda.stream(stream):
                dst.copy_(dev[i], non_blocking=True)
        pipe.run(7, None, lambda i, *r: b.__setitem__(i, r), fill_device=fill_device)
        for i in range(7):
            assert np.array_equal(a[i][0][1], b[i][0][1]) and a[i][0][1].shape[0] > 0
            assert len(a[i][2][1]) == len(b[i][2][1]) and all(np.array_equal(x, y) for x, y in zip(a[i][2][1], b[i][2][1]))
    finally:
        _cfg()


def test_test_net_with_device_jpeg_decode(tmp_path):
    """tools/test_net.py on a JSON roidb of per-frame .jpg files: TEST.DEVICE_JPEG_DECODE True runs end to end (clip assembly by
    utils/video.get_clip, nvJPEG decode on the loader threads, detections.pkl written)."""
    import cv2
    import json
    import pickle
    import subprocess
    import sys
    from detectandtrack_b200.ops import image_ops
    from test_gpu_tools import YAML, ROOT
    if not image_ops.jpeg_available():
        pytest.skip('nvJPEG is not installed on this machine')
    frames = tmp_path / 'vid0'
    frames.mkdir()
    entries = []
    for f in range(1, 5):
        p = str(frames / ('%06d.jpg' % f))
        cv2.imwrite(p, _image(96, 128, f), [cv2.IMWRITE_JPEG_QUALITY, 95])
        entries.append(dict(image=p, height=96, width=128, frame_id=f, flipped=False, id=f))
    js = tmp_path / 'frames.json'
    js.write_text(json.dumps(entries))
    cfgf = tmp_path / 'cfg.yaml'
    cfgf.write_text(YAML.replace('DATASET: synthetic_2x3_96x128', 'DATASET: %s' % js))
    res = {}
    for flag in ('False', 'True'):
        out = str(tmp_path / ('out_' + flag))
        r = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'test_net.py'), '--cfg', str(cfgf), 'OUTPUT_DIR', out,
                            'TEST.DEVICE_JPEG_DECODE', flag], env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        ddir = [os.path.join(dp, 'detections.pkl') for dp, _, fn in os.walk(out) if 'detections.pkl' in fn]
        res[flag] = pickle.load(open(ddir[0], 'rb'))
    assert len(res['True']['all_boxes'][1]) == len(res['False']['all_boxes'][1]) == 4
