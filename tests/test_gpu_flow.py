"""GPU: TRACKING.FLOW_SMOOTHING_ON on the device (csrc/flow.cu).

- dt_bgr_to_gray equals cv2.cvtColor bit for bit;
- dt_farneback_flow against live cv2.calcOpticalFlowFarneback on the textured pairs of tests/test_flow.py, several
  pairs per call: mean |d| <= 1e-3 px, p99.9 <= 1e-2 px, max <= 5e-2 px, and the median recovers a known translation
  to 0.01 px; against oracle/flow.py within the oracle-vs-cv2 bar;
- dt_flow_mean_abs equals np.abs(flow).mean() bit for bit;
- dt_flow_smooth_poses and _smooth_pose_video, fed the goldens' flows, equal the reference's goldens bit for bit;
- run_posetrack_tracking with FLOW_SMOOTHING_ON on a PNG video (known per-frame shifts, one cut) against the oracle
  pipeline with cv2's flow.
"""
import json
import os
import pickle

import numpy as np
import pytest

from oracle import flow as OF
from oracle import tracking as ot
from test_flow import ORACLE_MAX, ORACLE_P999, cv2_flow, golden_cases, textured_pair

pytestmark = pytest.mark.gpu

F32 = np.float32
MEAN_BAR, P999_BAR, MAX_BAR = 1e-3, 1e-2, 5e-2


def _bgr(gray):
    return np.repeat(gray[..., None], 3, axis=-1)


def _device_flows(pairs_of_frames):
    import torch
    from detectandtrack_b200.ops import flow_ops
    frames = []
    for a, b in pairs_of_frames:
        frames += [_bgr(a), _bgr(b)]
    d = torch.from_numpy(np.stack(frames)).cuda()
    out = flow_ops.farneback_flow(d, [(2 * i, 2 * i + 1) for i in range(len(pairs_of_frames))])
    return out


def test_gray_bit_exact_vs_cv2():
    import cv2
    import torch
    from detectandtrack_b200.ops import flow_ops
    bgr = np.random.RandomState(4).randint(0, 256, (3, 97, 131, 3)).astype(np.uint8)
    out = flow_ops.bgr_to_gray(torch.from_numpy(bgr).cuda()).cpu().numpy()
    assert np.array_equal(out, np.stack([cv2.cvtColor(f, cv2.COLOR_BGR2GRAY) for f in bgr]))


@pytest.mark.parametrize('kinds,h,w', [(('shift', 'patches'), 160, 240), (('zoom',), 161, 243),
                                       (('shift', 'zoom', 'patches'), 720, 1280)])
def test_flow_vs_cv2(kinds, h, w):
    pairs = [textured_pair(k, h, w, seed=i) for i, k in enumerate(kinds)]
    flows = _device_flows(pairs).cpu().numpy()
    for (a, b), k, f in zip(pairs, kinds, flows):
        ref = cv2_flow(a, b)
        d = np.abs(f - ref)
        stats = (float(d.mean()), float(np.percentile(d, 99.9)), float(d.max()))
        print('%s %dx%d: mean %.3g p99.9 %.3g max %.3g px' % ((k, h, w) + stats))
        assert stats[0] <= MEAN_BAR and stats[1] <= P999_BAR and stats[2] <= MAX_BAR, (k, stats)
        if k == 'shift':
            assert abs(np.median(f[..., 0]) - 1.75) < 0.01 and abs(np.median(f[..., 1]) + 0.6) < 0.01
        if h * w <= 161 * 243:
            o = np.abs(f - OF.farneback(a, b))
            assert o.max() <= ORACLE_MAX and np.percentile(o, 99.9) <= ORACLE_P999, (k, o.max())


@pytest.mark.parametrize('hw', [(160, 240), (161, 243), (720, 1280), (1080, 1920), (3, 5)])
def test_mean_abs_bit_exact(hw):
    import torch
    from detectandtrack_b200.ops import flow_ops
    rng = np.random.RandomState(hw[0])
    f = np.concatenate([rng.standard_normal((2,) + hw + (2,)) * s for s in (1.0, 7.0, 1e-3)]).astype(F32)
    out = flow_ops.flow_mean_abs(torch.from_numpy(f).cuda()).cpu().numpy()
    for i in range(len(f)):
        assert out[i].tobytes() == np.abs(f[i]).mean().tobytes(), (hw, i)


def test_smooth_poses_equals_goldens(golden):
    import torch
    from detectandtrack_b200.core import tracking_engine as te
    from detectandtrack_b200.ops import flow_ops
    for k, c in golden_cases(golden):
        N, ext, th = c['params']
        F = len(c['counts'])
        flows = [None if f is None else torch.from_numpy(f).cuda() for f in c['flows']] + [None]
        moves = [f is not None and not (np.abs(f).mean() > th) for f in c['flows']] + [False]
        out_t = te._output_tracks(c['track_lists'], c['counts'].tolist(), moves, int(N), bool(ext))
        oc = np.array([len(t) for t in out_t], np.int32)
        assert np.array_equal(oc, c['out_counts']), k
        omax = max(int(oc.max()), 1)
        ot_ = np.zeros((F, omax), np.int32)
        for f in range(F):
            ot_[f, :oc[f]] = out_t[f]
        is_start = np.zeros(F, np.uint8)
        is_start[0] = 1
        p, b = flow_ops.smooth_poses(c['poses'], c['boxes'], c['counts'], c['tracks'], is_start, flows,
                                     np.array([not m for m in moves], np.uint8), int(N), ot_, oc)
        p, b = p.cpu().numpy(), b.cpu().numpy()
        for f in range(F):
            n = oc[f]
            assert p[f, :n].tobytes() == c['out_poses'][f, :n].tobytes(), (k, f)
            assert b[f, :n].tobytes() == c['out_boxes'][f, :n].tobytes(), (k, f)


def test_smooth_pose_video_equals_goldens(golden, monkeypatch):
    import torch
    from detectandtrack_b200.core import tracking_engine as te
    from detectandtrack_b200.core.config import cfg, reset_cfg
    from detectandtrack_b200.ops import flow_ops
    try:
        for k, c in golden_cases(golden):
            N, ext, th = c['params']
            reset_cfg()
            cfg.TRACKING.FLOW_SMOOTHING_ON = True
            cfg.TRACKING.FLOW_SMOOTHING.N_CONTEXT_FRAMES = int(N)
            cfg.TRACKING.FLOW_SMOOTHING.EXTEND_TRACKS = bool(ext)
            cfg.TRACKING.FLOW_SMOOTHING.FLOW_SHOT_BOUNDARY_TH = float(th)
            dev = [None if f is None else torch.from_numpy(f).cuda() for f in c['flows']]
            means = [None if f is None else flow_ops.flow_mean_abs(f[None]).cpu().numpy()[0] for f in dev]
            monkeypatch.setattr(te, 'compute_optical_flow', lambda video, dev=dev, means=means: (dev, means))
            F = len(c['counts'])
            dets = {'all_boxes': [[], [b.copy() for b in c['box_lists']]], 'all_keyps': [[], [list(p) for p in c['pose_lists']]]}
            tracks = te._smooth_pose_video([({}, f) for f in range(F)], dets, c['track_lists'])
            for f in range(F):
                n = c['out_counts'][f]
                assert tracks[f] == c['out_tracks'][f, :n].tolist(), (k, f)
                b = dets['all_boxes'][1][f]
                assert b.dtype == (np.float64 if c['out_box_f64'][f] else F32) and b.shape == (n, 5), (k, f)
                assert b.tobytes() == c['out_boxes'][f, :n].astype(b.dtype).tobytes(), (k, f)
                ps = dets['all_keyps'][1][f]
                assert len(ps) == n and all(p.dtype == F32 and p.shape == (4, 17) for p in ps), (k, f)
                got = np.stack(ps) if n else np.zeros((0, 4, 17), F32)
                assert got.tobytes() == c['out_poses'][f, :n].tobytes(), (k, f)
    finally:
        reset_cfg()


# ---------------------------------------------------------------------------------------------------- end to end
SHIFTS = [(0, 0), (2, 1), (1, -1), (3, 0), (12, 12), (-1, 2), (2, 2)]      # per-frame shift; frame 4 is the cut


def _png_video(root, h=240, w=320):
    import cv2
    rng = np.random.RandomState(11)
    n = cv2.GaussianBlur(rng.rand(h + 96, w + 96, 3).astype(F32), (0, 0), 3)
    base = ((n - n.min()) / (n.max() - n.min()) * 255).astype(np.uint8)
    os.makedirs(os.path.join(root, 'vid'), exist_ok=True)
    paths, pos = [], np.zeros(2)
    for t, s in enumerate(SHIFTS):
        pos = pos + np.array(s)
        x0, y0 = 48 - int(pos[0]), 48 - int(pos[1])             # content moves by +shift
        p = os.path.join(root, 'vid', '%05d.png' % t)
        cv2.imwrite(p, base[y0:y0 + h, x0:x0 + w])
        paths.append(p)
    return paths


def _detections(rng, h=240, w=320):
    starts = np.array([[60, 50], [150, 70], [230, 90]], F32)
    boxes, poses, pos = [], [], np.zeros(2, F32)
    for t, s in enumerate(SHIFTS):
        pos = pos + np.array(s, F32)
        n = 3 if t != 2 else 2                                   # one person missing in frame 2
        b, ps = [], []
        for i in range(n):
            x, y = starts[i] + pos
            b.append([x - 20, y - 30, x + 20, y + 60, F32(0.95) + F32(0.01) * i])
            kx = np.floor(x - 15 + rng.uniform(0, 30, 17)) + F32(0.25)
            ky = np.floor(y - 25 + rng.uniform(0, 80, 17)) + F32(0.25)
            ps.append(np.stack([kx, ky, rng.normal(2, 2, 17), rng.uniform(0, 1, 17)]).astype(F32))
        boxes.append(np.array(b, F32))
        poses.append(ps)
    return {'all_boxes': [[], boxes], 'all_keyps': [[], poses]}


def test_run_posetrack_tracking_with_flow_smoothing_vs_oracle(tmp_path):
    import cv2
    from detectandtrack_b200.core import tracking_engine as te
    from detectandtrack_b200.core.config import cfg, reset_cfg
    paths = _png_video(str(tmp_path / 'frames'))
    dets = _detections(np.random.RandomState(5))
    json_data = [{'image': p, 'height': 240, 'width': 320} for p in paths]
    out_dir = str(tmp_path / 'out')
    os.makedirs(out_dir)
    with open(os.path.join(out_dir, 'detections.pkl'), 'wb') as f:
        pickle.dump(dets, f)
    N = 2
    reset_cfg()
    try:
        cfg.KRCNN.NUM_KEYPOINTS = 17
        cfg.TRACKING.FLOW_SMOOTHING_ON = True
        cfg.TRACKING.FLOW_SMOOTHING.N_CONTEXT_FRAMES = N
        out = te.run_posetrack_tracking(out_dir, json_data, write_json=True)
        th = cfg.TRACKING.FLOW_SMOOTHING.FLOW_SHOT_BOUNDARY_TH
        conf = cfg.TRACKING.CONF_FILTER_INITIAL_DETS
    finally:
        reset_cfg()
    # oracle pipeline: prune, link, cv2 flow, smoothing
    boxes, poses = [], []
    for t in range(len(paths)):
        b = dets['all_boxes'][1][t].copy()
        sel = ot.prune_boxes(b, 240, 320, conf)
        boxes.append(b[sel])
        poses.append([dets['all_keyps'][1][t][i] for i in sel])
    tracks = ot.compute_tracks_video(boxes, solver='scipy')
    grays = [cv2.cvtColor(cv2.imread(p), cv2.COLOR_BGR2GRAY) for p in paths]
    flows = [cv2_flow(grays[q], grays[q + 1]) for q in range(len(paths) - 1)]
    assert np.abs(flows[3]).mean() > th and all(np.abs(f).mean() <= th for i, f in enumerate(flows) if i != 3)
    rp, rb, rt = OF.smooth_pose_video(poses, boxes, [list(map(int, t)) for t in tracks], flows, N, True, th)
    for t in range(len(paths)):
        assert out['all_tracks'][1][t] == rt[t], t
        b = out['all_boxes'][1][t]
        assert b.dtype == rb[t].dtype and np.array_equal(b, rb[t]), t
        p, r = np.stack(out['all_keyps'][1][t]), np.stack(rp[t])
        assert np.array_equal(p[:, 2:], r[:, 2:]), t                   # scores and row 3: identical
        assert np.abs(p[:, :2] - r[:, :2]).max() <= N * MAX_BAR, t      # positions: within N lookups of the flow bar
    with open(os.path.join(out_dir, 'detections_withTracks.pkl'), 'rb') as f:
        saved = pickle.load(f)
    assert saved['all_tracks'][1] == out['all_tracks'][1]
    jdir = os.path.join(out_dir, 'detections_withTracks.pkl_json')
    files = [os.path.join(jdir, n) for n in os.listdir(jdir)]
    assert files and all(json.load(open(p)) for p in files)
