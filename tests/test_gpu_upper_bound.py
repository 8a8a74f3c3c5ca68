"""GPU: the upper-bound experiments against the reference's own code (tests/golden/upper_bound.npz): the tracking modes
TRACKING.DEBUG.UPPER_BOUND / _2_GT_KPS / _2_GT_KPS_ONLY_CONF / _5_GT_KPS_ONLY (kept rows, boxes, poses and track ids
bit-equal, pose-pck weight 0 and 1, hungarian and greedy) and poseval's upper-bound MOT (-u)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Z = np.load(os.path.join(ROOT, 'tests', 'golden', 'upper_bound.npz'))
P = np.load(os.path.join(ROOT, 'tests', 'golden', 'poseval.npz'))
N_CASES = len({k.split('_')[0] for k in Z.files if k.startswith('t')})
N_MODES = len({k.split('_')[1] for k in Z.files if k.startswith('t0_m')})


def _inputs(t):
    g = lambda n: Z['t%d_%s' % (t, n)]
    counts, gcounts = g('counts'), g('gt_counts')
    dets = {'all_boxes': [[], [g('boxes')[f, :n].copy() for f, n in enumerate(counts)]],
            'all_keyps': [[], [[g('poses')[f, i].copy() for i in range(n)] for f, n in enumerate(counts)]]}
    json_data = [{'image': 'vid/%05d.jpg' % f, 'boxes': g('gt_boxes')[f, :n].copy(), 'gt_keypoints': g('gt_kps')[f, :n].copy(),
                  'tracks': g('gt_tracks')[f, :n].copy()} for f, n in enumerate(gcounts)]
    return json_data, dets


@pytest.mark.parametrize('t', range(N_CASES))
@pytest.mark.parametrize('m', range(N_MODES))
def test_tracking_modes_vs_reference(t, m):
    from detectandtrack_b200.core import tracking_engine as te
    from detectandtrack_b200.core.config import cfg, reset_cfg
    reset_cfg()
    ub, ub2, conf, ub5, w, greedy = Z['t%d_m%d_params' % (t, m)]
    d = cfg.TRACKING.DEBUG
    d.UPPER_BOUND, d.UPPER_BOUND_2_GT_KPS, d.UPPER_BOUND_2_GT_KPS_ONLY_CONF, d.UPPER_BOUND_5_GT_KPS_ONLY = \
        bool(ub), bool(ub2), bool(conf), bool(ub5)
    cfg.TRACKING.DISTANCE_METRICS = ('bbox-overlap', 'cnn-cosdist', 'pose-pck')
    cfg.TRACKING.DISTANCE_METRIC_WTS = (1.0, 0.0, float(w))
    cfg.TRACKING.BIPARTITE_MATCHING_ALGO = 'greedy' if greedy else 'hungarian'
    try:
        json_data, dets = _inputs(t)
        te.compute_matches_tracks(json_data, dets)
        pre = 't%d_m%d_' % (t, m)
        counts = Z[pre + 'out_counts']
        for f, n in enumerate(counts):
            b = dets['all_boxes'][1][f]
            assert b.shape == (n, 5) and b.dtype == np.float32, (f, b.shape)
            assert np.array_equal(b.view(np.int32), Z[pre + 'out_boxes'][f, :n].view(np.int32)), f
            p = dets['all_keyps'][1][f]
            assert len(p) == n
            for i in range(n):
                assert p[i].dtype == np.float32
                assert np.array_equal(p[i].view(np.int32), Z[pre + 'out_poses'][f, i].view(np.int32)), (f, i)
            assert dets['all_tracks'][1][f] == Z[pre + 'out_tracks'][f, :n].tolist(), f
    finally:
        reset_cfg()


def _dirs(case, tmp):
    from detectandtrack_b200.datasets import posetrack_synth as S
    files = json.loads(str(P[case + '/files']))
    return S.write_dirs({n: (files['gt'][n], files['pred'][n]) for n in files['gt']}, str(tmp))


@pytest.mark.parametrize('case', ['edge', 'synth', 'val3'])
def test_poseval_upper_bound_vs_reference(case, tmp_path):
    from detectandtrack_b200.datasets import posetrack_eval as E
    gt_dir, pred_dir = _dirs(case, tmp_path)
    gtFramesAll, prFramesAll, names = E.load_data_dir(gt_dir, pred_dir)
    res = E.evaluate_pack(E.PoseTrackPack(gtFramesAll, prFramesAll, names), True, True, per_video=True, track_upper_bound=True)
    n = len(Z['u_%s/seq_counts' % case])
    assert np.array_equal(res['raw']['counts'][:n].astype(np.int64), Z['u_%s/seq_counts' % case])
    np.testing.assert_allclose(res['raw']['sumd'][:n], Z['u_%s/seq_sumd' % case], rtol=1e-12, atol=0)
    np.testing.assert_allclose(res['metrics'], Z['u_%s/metrics' % case], rtol=1e-12, atol=0)
    # AP is the normal assignment's
    np.testing.assert_allclose(res['ap'][0], P[case + '/apAll'], rtol=1e-12, atol=0)
    # evaluate_upper_bound is the same path; evaluate() keeps the upper bound out
    (ap, _, _), metrics = E.evaluate_upper_bound(gt_dir, pred_dir, verbose=False)
    np.testing.assert_allclose(metrics, Z['u_%s/metrics' % case], rtol=1e-12, atol=0)


def test_eval_posetrack_cli_upper_bound(tmp_path):
    from detectandtrack_b200.datasets import posetrack_eval as E
    gt_dir, pred_dir = _dirs('synth', tmp_path)
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'eval_posetrack.py'), '-g', gt_dir, '-p', pred_dir, '-t', '-u'],
                       env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert E.get_mot_header() in r.stdout
    assert E.get_format_row(E.get_cum(Z['u_synth/metrics'])) in r.stdout


def test_run_eval_upper_bound_key(tmp_path):
    from detectandtrack_b200.core import mpii_eval_engine as M
    from detectandtrack_b200.core.config import cfg, reset_cfg
    gt_dir, pred_dir = _dirs('synth', tmp_path)
    reset_cfg()
    try:
        cfg.TRACKING.DEBUG.UPPER_BOUND_4_EVAL_UPPER_BOUND = True
        ap, mota = M._run_eval(gt_dir, pred_dir, eval_tracking=True)
    finally:
        reset_cfg()
    assert mota == pytest.approx(Z['u_synth/metrics'][-4, 0], rel=1e-12)
    assert ap == pytest.approx(P['synth/apAll'][-1, 0], rel=1e-12)
