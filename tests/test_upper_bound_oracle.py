"""CPU: the upper-bound oracle (tests/upper_bound_oracle.py) reproduces the reference's own results
(tests/golden/upper_bound.npz): every tracking case and mode bit-exactly, poseval's upper-bound MOT counts exactly and
MOTA / sumD to 1e-12."""
import json
import os

import numpy as np
import pytest

import upper_bound_oracle as U
from detectandtrack_b200.datasets import posetrack_synth as S
from oracle import poseval as ope

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Z = np.load(os.path.join(ROOT, 'tests', 'golden', 'upper_bound.npz'))
P = np.load(os.path.join(ROOT, 'tests', 'golden', 'poseval.npz'))
N_CASES = len({k.split('_')[0] for k in Z.files if k.startswith('t')})
N_MODES = len({k.split('_')[1] for k in Z.files if k.startswith('t0_m')})


def golden_frames(t):
    g = lambda n: Z['t%d_%s' % (t, n)]
    return [dict(boxes=g('boxes')[f, :n].copy(), poses=[g('poses')[f, i].copy() for i in range(n)],
                 gt_boxes=g('gt_boxes')[f, :G].copy(), gt_kps=g('gt_kps')[f, :G].copy(), gt_tracks=g('gt_tracks')[f, :G].copy())
            for f, (n, G) in enumerate(zip(g('counts'), g('gt_counts')))]


@pytest.mark.parametrize('t', range(N_CASES))
def test_tracking_oracle_vs_reference(t):
    for m in range(N_MODES):
        pre = 't%d_m%d_' % (t, m)
        ub, ub2, conf, ub5, w, greedy = Z[pre + 'params']
        b, p, tr = U.compute_tracks_video(golden_frames(t), bool(ub), bool(ub2), bool(conf), bool(ub5), 1.0, float(w),
                                          'greedy' if greedy else 'hungarian')
        for f, n in enumerate(Z[pre + 'out_counts']):
            assert b[f].shape == (n, 5) and b[f].dtype == np.float32, (m, f)
            assert np.array_equal(b[f].view(np.int32), Z[pre + 'out_boxes'][f, :n].view(np.int32)), (m, f)
            assert len(p[f]) == n
            for i in range(n):
                assert np.array_equal(p[f][i].astype(np.float32).view(np.int32), Z[pre + 'out_poses'][f, i].view(np.int32)), (m, f, i)
            assert tr[f] == Z[pre + 'out_tracks'][f, :n].tolist(), (m, f)


@pytest.mark.parametrize('case', ['edge', 'synth', 'val3'])
def test_poseval_upper_bound_oracle_vs_reference(case, tmp_path):
    files = json.loads(str(P[case + '/files']))
    gt_dir, pred_dir = S.write_dirs({n: (files['gt'][n], files['pred'][n]) for n in files['gt']}, str(tmp_path))
    gt, pr, _ = ope.load_data_dir(gt_dir, pred_dir)
    metrics, per_seq = U.evaluate_tracking_upper_bound(gt, pr)
    assert np.array_equal(np.array([c for c, _ in per_seq], np.int64), Z['u_%s/seq_counts' % case])
    np.testing.assert_allclose(np.array([d for _, d in per_seq]), Z['u_%s/seq_sumd' % case], rtol=1e-12, atol=0)
    np.testing.assert_allclose(metrics, Z['u_%s/metrics' % case], rtol=1e-12, atol=0)
