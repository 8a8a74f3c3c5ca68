"""CPU: the upper-bound experiments' host rejections (before any device work) and the C ABI argument checks of their
kernels; the goldens' consistency with the reference's rules."""
import os

import numpy as np
import pytest

from detectandtrack_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Z = np.load(os.path.join(ROOT, 'tests', 'golden', 'upper_bound.npz'))


@pytest.fixture
def ub_cfg():
    from detectandtrack_b200.core.config import cfg, reset_cfg
    reset_cfg()
    yield cfg
    reset_cfg()


def _dets(n_frames=3, T=1):
    return {'all_boxes': [[], [np.array([[10, 10, 80, 90] * T + [0.9]], np.float32) for _ in range(n_frames)]],
            'all_keyps': [[], [[np.zeros((4, 17), np.float32)] for _ in range(n_frames)]]}


def _roidb(n_frames=3, gt=True, gt_cols=4):
    out = []
    for f in range(n_frames):
        e = {'image': 'v/%05d.jpg' % f, 'height': 100, 'width': 100}
        if gt:
            e.update(boxes=np.zeros((1, gt_cols), np.float32), gt_keypoints=np.zeros((1, 3, 17), np.int32), tracks=np.array([4]))
        out.append(e)
    return out


@pytest.mark.parametrize('key', ['UPPER_BOUND', 'UPPER_BOUND_5_GT_KPS_ONLY'])
def test_roidb_without_gt_is_rejected(ub_cfg, key):
    from detectandtrack_b200.core import tracking_engine as te
    setattr(ub_cfg.TRACKING.DEBUG, key, True)
    with pytest.raises(ValueError, match="no ground truth 'boxes'"):
        te.compute_matches_tracks(_roidb(gt=False), _dets())


def test_three_shots_is_rejected(ub_cfg):
    from detectandtrack_b200.core import tracking_engine as te
    ub_cfg.TRACKING.DEBUG.UPPER_BOUND_3_SHOTS = True
    with pytest.raises(NotImplementedError, match='shot_boundaries_val.csv'):
        te.compute_matches_tracks(_roidb(), _dets())


def test_gt_and_detection_frame_counts_must_agree(ub_cfg):
    from detectandtrack_b200.core import tracking_engine as te
    ub_cfg.TRACKING.DEBUG.UPPER_BOUND = True
    with pytest.raises(NotImplementedError, match='GT boxes of 4 columns for detections of 3 frame'):
        te.compute_matches_tracks(_roidb(), _dets(T=3))


def test_gt_kps_needs_centre_frame_boxes(ub_cfg):
    from detectandtrack_b200.core import tracking_engine as te
    ub_cfg.TRACKING.DEBUG.UPPER_BOUND = True
    ub_cfg.TRACKING.DEBUG.UPPER_BOUND_2_GT_KPS = True
    with pytest.raises(NotImplementedError, match='T = 3'):
        te.compute_matches_tracks(_roidb(gt_cols=12), _dets(T=3))


def test_golden_tracks_are_gt_tracks():
    """Under UPPER_BOUND every kept detection carries a track id of its frame's GT, and _5 alone keeps every row."""
    cases = sorted({k.split('_')[0] for k in Z.files if k.startswith('t')})
    for t in cases:
        modes = sorted({k.split('_')[1] for k in Z.files if k.startswith(t + '_m')})
        for m in modes:
            pre = '%s_%s_' % (t, m)
            ub, ub2, conf, ub5, w, greedy = Z[pre + 'params']
            for f, n in enumerate(Z[pre + 'out_counts']):
                gt = set(Z[t + '_gt_tracks'][f, :Z[t + '_gt_counts'][f]].tolist())
                tr = Z[pre + 'out_tracks'][f, :n].tolist()
                if ub:
                    assert set(tr) <= gt and n == min(Z[t + '_counts'][f], len(gt))
                else:
                    assert n == Z[t + '_counts'][f]


def test_capi_argument_checks():
    cases = [
        ('dt_gt_frame_costs', (None, 5, 1, None, 4, 17, 2, 1, 0.5, None, 2, 225, 1.0, 0.0, None, None), b'dmax=225'),
        ('dt_gt_frame_costs', (None, 5, 1, None, 4, 17, 2, 1, 0.5, None, 2, 8, 1.0, 1.0, None, None), b'pose-pck'),
        ('dt_gt_frame_costs', (None, 5, 1, None, 4, 17, 2, 1, 0.5, None, 2, 8, 1.0, 0.0, None, None), b'null pointer'),
        ('dt_track_upper_bound', (None, 5, None, 4, 17, None, None, 2, 225, None, 0, None, 0, 0, None, None, None, None, None),
         b'dmax=225'),
        ('dt_track_upper_bound', (None, 5, None, 2, 17, None, None, 2, 8, None, 0, None, 0, 0, None, None, None, None, None),
         b'R=2'),
        ('dt_track_upper_bound', (None, 5, None, 4, 17, None, None, 2, 8, None, 0, None, 0, 2, None, None, None, None, None),
         b'bad flags 2'),
        ('dt_track_upper_bound', (None, 5, None, 4, 17, None, None, 2, 8, None, 0, None, 0, 1, None, None, None, None, None),
         b'COMPACT needs matches'),
        ('dt_posetrack_upper_bound', (None, None, None, 4, None, None, None, None, None, 65, 10) + (None,) * 6, b'max_gt=65'),
        ('dt_posetrack_upper_bound', (None, None, None, 4, None, None, None, None, None, 10, 225) + (None,) * 6, b'max_pr=225'),
        ('dt_posetrack_upper_bound', (None, None, None, 4, None, None, None, None, None, 10, 10) + (None,) * 6, b'null pointer'),
    ]
    lib = L.lib()
    for name, args, msg in cases:
        rc = getattr(lib, name)(*args)
        assert rc != 0, name
        assert msg in lib.dt_last_error(), (name, lib.dt_last_error())
    # empty batches are no-ops
    assert lib.dt_gt_frame_costs(None, 5, 1, None, 4, 17, 2, 1, 0.5, None, 0, 8, 1.0, 0.0, None, None) == 0
    assert lib.dt_posetrack_upper_bound(None, None, None, 0, None, None, None, None, None, 0, 0, *(None,) * 6) == 0


def test_evaluate_keeps_the_upper_bound_out():
    from detectandtrack_b200.datasets import posetrack_eval as E
    with pytest.raises(NotImplementedError, match='evaluate_upper_bound'):
        E.evaluate('/nonexistent', '/nonexistent', eval_upper_bound=True)
