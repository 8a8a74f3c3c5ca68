"""CPU: TRACKING.FLOW_SMOOTHING_ON without a GPU.

- oracle/flow.py's smoothing equals the reference's own _smooth_pose_video (tests/golden/flow_smooth.npz) bit for bit,
  and the tracking engine's host-side track order equals the reference's list(set(...)) order;
- oracle/flow.py's Farneback equals cv2.calcOpticalFlowFarneback stage by stage and end to end, on textured pairs under
  a translation, a zoom plus rotation and independently moving patches (measured: max |d| 3.4e-5 px at 720x1280);
- the np.abs(flow).mean() restatement is numpy's, bit for bit;
- the host rejects what the device path does not run before any CUDA call, and the new C entry points check their
  arguments on the host.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import flow as OF

F32 = np.float32
# oracle vs cv2 on the textured pairs below (cv2 4.13, SIMD + IPP build): measured max 3.4e-5 px, p99.9 1.5e-5 px
ORACLE_MAX, ORACLE_P999 = 1e-4, 5e-5


def golden_cases(golden):
    g = golden('flow_smooth')
    k = 0
    while 'c%d_params' % k in g:
        c = {n[len('c%d_' % k):]: g[n] for n in g if n.startswith('c%d_' % k)}
        F = len(c['counts'])
        cnt = c['counts']
        c['pose_lists'] = [[c['poses'][f, i] for i in range(cnt[f])] for f in range(F)]
        c['box_lists'] = [c['boxes'][f, :cnt[f]] for f in range(F)]
        c['track_lists'] = [c['tracks'][f, :cnt[f]].tolist() for f in range(F)]
        c['flows'] = [None if c['flow_none'][q] else c['flow%d' % q] for q in range(F - 1)]
        yield k, c
        k += 1


def test_oracle_smoothing_equals_reference_goldens(golden):
    n = 0
    for k, c in golden_cases(golden):
        N, ext, th = c['params']
        p, b, t = OF.smooth_pose_video(c['pose_lists'], c['box_lists'], c['track_lists'], c['flows'], int(N), bool(ext), th)
        oc = c['out_counts']
        for f in range(len(oc)):
            assert t[f] == c['out_tracks'][f, :oc[f]].tolist(), (k, f)
            assert all(x.dtype == F32 for x in p[f])
            assert np.array_equal(np.stack(p[f]) if oc[f] else np.zeros((0, 4, 17), F32), c['out_poses'][f, :oc[f]]), (k, f)
            assert b[f].dtype == (np.float64 if c['out_box_f64'][f] else F32), (k, f)
            assert np.array_equal(b[f], c['out_boxes'][f, :oc[f]]), (k, f)
        n += 1
    assert n >= 20


def test_host_track_order_equals_reference(golden):
    from detectandtrack_b200.core import tracking_engine as te
    unsorted = 0
    for k, c in golden_cases(golden):
        N, ext, th = c['params']
        moves = [f is not None and not (np.abs(f).mean() > th) for f in c['flows']] + [False]
        out = te._output_tracks(c['track_lists'], c['counts'].tolist(), moves, int(N), bool(ext))
        oc = c['out_counts']
        for f in range(len(oc)):
            assert out[f] == c['out_tracks'][f, :oc[f]].tolist(), (k, f)
            unsorted += out[f] != sorted(out[f]) and bool(ext)
    assert unsorted > 0, 'no case where the set order differs from the sorted order'


# ---------------------------------------------------------------------------------------------------- Farneback
def _texture(rng, h, w, sigma=3.0):
    import cv2
    n = rng.rand(h, w).astype(F32)
    n = cv2.GaussianBlur(n, (0, 0), sigma)
    return (n - n.min()) / (n.max() - n.min()) * F32(255)


def textured_pair(kind, h, w, seed=0):
    """Two uint8 gray frames: low-passed noise under a known translation (1.75, -0.6) px, a zoom plus rotation, or
    independently moving patches."""
    import cv2
    rng = np.random.RandomState(seed)
    base = _texture(rng, h + 64, w + 64)
    if kind == 'shift':
        M = np.float32([[1, 0, 1.75], [0, 1, -0.6]])
    elif kind == 'zoom':
        M = cv2.getRotationMatrix2D(((w + 64) / 2, (h + 64) / 2), 3, 1.04).astype(F32)
    else:
        M = np.float32([[1, 0, 0.5], [0, 1, 0.25]])
    moved = cv2.warpAffine(base, M, (w + 64, h + 64), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_REFLECT)
    if kind == 'patches':
        for i, (dy, dx) in enumerate([(3, -2), (-2, 4), (1, 1)]):
            y0, x0 = 16 + (i * h) // 4, 16 + (i * w) // 4
            ph, pw = h // 4, w // 4
            moved[y0 + dy:y0 + dy + ph, x0 + dx:x0 + dx + pw] = base[y0:y0 + ph, x0:x0 + pw]
    a, b = base[32:32 + h, 32:32 + w], moved[32:32 + h, 32:32 + w]
    return np.clip(a, 0, 255).astype(np.uint8), np.clip(b, 0, 255).astype(np.uint8)


def cv2_flow(a, b):
    import cv2
    return cv2.calcOpticalFlowFarneback(a, b, None, 0.5, 10, min(a.shape[:2]) // 5, 10, 7, 1.5, cv2.OPTFLOW_FARNEBACK_GAUSSIAN)


def test_gray_conversion_equals_cv2():
    import cv2
    bgr = np.random.RandomState(1).randint(0, 256, (37, 53, 3)).astype(np.uint8)
    assert np.array_equal(OF.bgr_to_gray(bgr), cv2.cvtColor(bgr, cv2.COLOR_BGR2GRAY))


@pytest.mark.parametrize('hw', [(160, 240), (161, 243)])
def test_pyramid_stages_equal_cv2(hw):
    import cv2
    h, w = hw
    img = textured_pair('zoom', h, w)[0].astype(F32)
    levels = OF.level_sizes(h, w)
    assert [lv[0] for lv in levels] == [2, 1, 0]             # levels=10 stops at the 32-px floor
    for lv, s, ww, hh, ks, sigma in levels:
        ref = cv2.GaussianBlur(img, (ks, ks), sigma, sigma)
        assert np.abs(OF.gaussian_blur(img, ks, sigma) - ref).max() <= 1e-4, lv
        assert np.abs(OF.resize_linear(ref, ww, hh) - cv2.resize(ref, (ww, hh), interpolation=cv2.INTER_LINEAR)).max() <= 5e-4
    flow = np.random.RandomState(2).normal(0, 2, (h // 2, w // 2, 2)).astype(F32)
    assert np.abs(OF.resize_linear(flow, w, h) - cv2.resize(flow, (w, h), interpolation=cv2.INTER_LINEAR)).max() <= 1e-5


@pytest.mark.parametrize('kind,h,w', [('shift', 160, 240), ('zoom', 161, 243), ('patches', 160, 240),
                                      ('shift', 720, 1280)])
def test_oracle_farneback_equals_cv2(kind, h, w):
    a, b = textured_pair(kind, h, w)
    ref = cv2_flow(a, b)
    d = np.abs(OF.farneback(a, b) - ref)
    assert d.max() <= ORACLE_MAX and np.percentile(d, 99.9) <= ORACLE_P999, (d.max(), np.percentile(d, 99.9))
    if kind == 'shift':
        assert abs(np.median(ref[..., 0]) - 1.75) < 0.01 and abs(np.median(ref[..., 1]) + 0.6) < 0.01


@pytest.mark.parametrize('shape', [(160, 240, 2), (161, 243, 2), (720, 1280, 2), (1080, 1920, 2), (3, 5, 2), (8, 8, 2)])
def test_mean_abs_restatement_equals_numpy(shape):
    rng = np.random.RandomState(sum(shape))
    for scale in (1.0, 7.0, 1e-3):
        f = (rng.standard_normal(shape) * scale).astype(F32)
        ref = np.abs(f).mean()
        assert ref.dtype == F32
        assert OF.flow_mean_abs(f).tobytes() == ref.tobytes(), (shape, scale)


# ---------------------------------------------------------------------------------------------------- host checks
def _dets(T=1, K=17):
    boxes = [np.array([[10, 10, 50, 80] * T + [0.99]], F32), np.array([[12, 11, 52, 81] * T + [0.98]], F32)]
    poses = [[np.zeros((4, K), F32)], [np.zeros((4, K), F32)]]
    json_data = [{'image': 'v/%d.jpg' % i, 'height': 100, 'width': 100} for i in range(2)]
    return {'all_boxes': [[], boxes], 'all_keyps': [[], poses]}, json_data


@pytest.mark.parametrize('what', ['T3', 'K15', 'combine', 'lstm', 'context'])
def test_host_rejections_before_any_cuda_call(what, tmp_path):
    import pickle
    from detectandtrack_b200.core import tracking_engine as te
    from detectandtrack_b200.core.config import cfg, reset_cfg
    reset_cfg()
    try:
        cfg.TRACKING.FLOW_SMOOTHING_ON = True
        dets, json_data = _dets(T=3 if what == 'T3' else 1, K=15 if what == 'K15' else 17)
        if what == 'combine':
            cfg.TRACKING.DEBUG.FLOW_SMOOTHING_COMBINE = True
        if what == 'lstm':
            cfg.TRACKING.FLOW_SMOOTHING_ON = False
            cfg.TRACKING.LSTM_TEST.LSTM_TRACKING_ON = True
        if what == 'context':
            cfg.TRACKING.FLOW_SMOOTHING.N_CONTEXT_FRAMES = 17
        # without a GPU the first device call raises RuntimeError: NotImplementedError means nothing reached the device
        with pytest.raises(NotImplementedError):
            te.compute_matches_tracks(json_data, dets, None)
        with open(str(tmp_path / 'detections.pkl'), 'wb') as f:
            pickle.dump(dets, f)
        cfg.TRACKING.KEEP_CENTER_DETS_ONLY = False
        with pytest.raises(NotImplementedError):
            te.run_posetrack_tracking(str(tmp_path), json_data, write_json=False)
    finally:
        reset_cfg()


def _abi_cases():
    from detectandtrack_b200 import _lib as L
    sz = C.c_size_t(0)
    one = (C.c_int * 2)(0, 1)
    return [
        ('dt_bgr_to_gray', (None, -1, None, None), b'npix'),
        ('dt_bgr_to_gray', (None, 10, None, None), b'null'),
        ('dt_farneback_workspace_bytes', (0, 10, 2, 1, C.byref(sz)), b'bad args'),
        ('dt_farneback_flow', (None, 2, 0, 10, None, 1, 0.5, 10, 3, 10, 7, 1.5, 256, None, None, 0, None), b'bad shape'),
        ('dt_farneback_flow', (None, 2, 64, 64, None, 1, 1.5, 10, 12, 10, 7, 1.5, 256, None, None, 0, None), b'pyr_scale'),
        ('dt_farneback_flow', (None, 2, 64, 64, None, 1, 0.5, 10, 12, 10, 6, 1.5, 256, None, None, 0, None), b'poly_n'),
        ('dt_farneback_flow', (None, 2, 64, 64, None, 1, 0.5, 10, 12, 10, 7, 1.5, 0, None, None, 0, None), b'GAUSSIAN'),
        ('dt_farneback_flow', (None, 2, 64, 64, None, 1, 0.5, 10, 400, 10, 7, 1.5, 256, None, None, 0, None), b'winsize'),
        ('dt_farneback_flow', (one, 2, 64, 64, one, 1, 0.5, 10, 12, 10, 7, 1.5, 256, one, one, 16, None), b'workspace'),
        ('dt_flow_mean_abs', (None, 1, 0, 4, None, None), b'bad shape'),
        ('dt_flow_mean_abs', (one, 1, 4096, 4096, one, None), b'exceed'),
        ('dt_flow_smooth_poses', (None, None, None, None, None, 2, 4, 17, None, None, None, 17, None, None, 4, None, None, None),
         b'n_context'),
        ('dt_flow_smooth_poses', (None, None, None, None, None, 2, 0, 17, None, None, None, 1, None, None, 4, None, None, None),
         b'bad shape'),
        ('dt_flow_smooth_poses', (one, one, one, one, one, 2, 4, 17, None, None, None, 1, one, one, 4, one, one, None),
         b'needs the flows'),
    ]


@pytest.mark.parametrize('i', range(14))
def test_entry_points_reject_bad_arguments_without_a_gpu(i):
    from detectandtrack_b200 import _lib as L
    name, args, msg = _abi_cases()[i]
    lib = L.lib()
    rc = getattr(lib, name)(*args)
    assert rc != 0, name
    assert msg in lib.dt_last_error(), (name, lib.dt_last_error())


def test_workspace_query_is_host_only():
    from detectandtrack_b200 import _lib as L
    a, b = C.c_size_t(0), C.c_size_t(0)
    L.call('dt_farneback_workspace_bytes', 720, 1280, 2, 1, C.byref(a))
    L.call('dt_farneback_workspace_bytes', 720, 1280, 3, 2, C.byref(b))
    assert 0 < a.value < b.value


def test_read_key_frame_is_the_clip_centre(tmp_path):
    import cv2
    from detectandtrack_b200.core import test_engine, tracking_engine as te
    from detectandtrack_b200.core.config import cfg, reset_cfg
    reset_cfg()
    try:
        cfg.MODEL.VIDEO_ON, cfg.VIDEO.NUM_FRAMES = True, 3
        syn = {'synthetic': True, 'height': 24, 'width': 40, 'seed': 7}
        assert np.array_equal(te.read_key_frame(syn), test_engine.read_image_video(syn)[1])
    finally:
        reset_cfg()
    paths = []
    for i in range(3):
        paths.append(str(tmp_path / ('%d.png' % i)))
        cv2.imwrite(paths[-1], np.full((8, 10, 3), 40 * i, np.uint8))
    assert np.array_equal(te.read_key_frame({'image': paths}), cv2.imread(paths[1]))
    assert np.array_equal(te.read_key_frame({'image': paths[2]}), cv2.imread(paths[2]))
