"""GPU: tools/compute_tracks.py end to end with the flags of each README upper-bound command, on a JSON-list roidb with GT
(plain JSON lists, float keypoint coordinates) and EVAL.POSETRACK_ANNOTATION_DIR: the tracked detections equal the CPU
oracle (tests/upper_bound_oracle.py) bit for bit, and the (total mAP, total MOTA) it logs is the oracle's score of the
JSON files it wrote."""
import json
import os
import pickle
import re
import subprocess
import sys

import numpy as np
import pytest

import upper_bound_oracle as U
from oracle import poseval as ope

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K = 17
H, W = 480, 640
README = {
    'perfect tracking': ['TRACKING.DEBUG.UPPER_BOUND_4_EVAL_UPPER_BOUND', 'True'],
    'perfect keypoints': ['TRACKING.DEBUG.UPPER_BOUND_5_GT_KPS_ONLY', 'True'],
    'both': ['TRACKING.DEBUG.UPPER_BOUND_5_GT_KPS_ONLY', 'True', 'TRACKING.DEBUG.UPPER_BOUND_4_EVAL_UPPER_BOUND', 'True'],
    'GT tracks and keypoints': ['TRACKING.DEBUG.UPPER_BOUND_2_GT_KPS', 'True'],
}
YAML = '''
MODEL:
  TYPE: keypoint_rcnn
KRCNN:
  NUM_KEYPOINTS: 17
EVAL:
  EVAL_MPII_DROP_DETECTION_THRESHOLD: 0.0
TEST:
  DATASET: %s
'''


def _world(root, videos=2, frames=6, people=4, seed=11):
    """roidb.json (GT per frame), detections.pkl (jittered GT, a false positive per frame) and the PoseTrack GT files."""
    from detectandtrack_b200.core import mpii_eval_engine as M
    rng = np.random.RandomState(seed)
    roidb, boxes, poses, annot = [], [], [], os.path.join(root, 'annot')
    os.makedirs(annot)
    for v in range(videos):
        c = rng.uniform([120, 150], [W - 120, H - 150], (people, 2))
        annolist = []
        for f in range(frames):
            c = c + rng.normal(0, 4, c.shape)
            gb = np.concatenate([c - [40, 90], c + [40, 90]], 1)
            kp = np.zeros((people, 3, K))
            kp[:, 0] = c[:, :1] + rng.uniform(-35, 35, (people, K)) + 0.4
            kp[:, 1] = c[:, 1:] + rng.uniform(-85, 85, (people, K)) + 0.7
            kp[:, 2] = 2
            tracks = [10 * v + t for t in range(people)]
            name = 'vid%03d/%06d.jpg' % (v, f + 1)
            roidb.append({'image': name, 'height': H, 'width': W, 'frame_id': f + 1, 'boxes': gb.tolist(),
                          'gt_keypoints': kp.tolist(), 'tracks': tracks})
            order = rng.permutation(people)
            db = np.hstack([gb[order] + rng.normal(0, 6, (people, 4)), rng.uniform(0.95, 1, (people, 1))])
            db = np.vstack([db, [20, 20, 90, 150, 0.97]]).astype(np.float32)
            dp = np.zeros((people + 1, 4, K), np.float32)
            dp[:people, :2] = kp[order, :2] + rng.normal(0, 6, (people, 2, K))
            dp[:, 2] = rng.uniform(1, 3, (people + 1, K))
            dp[:, 3] = rng.uniform(0, 1, (people + 1, K))
            dp[people, :2] = [[40] * K, [60] * K]
            boxes.append(db)
            poses.append(list(dp))
            rects = []
            for t in range(people):
                pts = []
                for j, dst in enumerate(M.dst_keypoints):
                    s = M.posetrack_src_keypoints.index('head_bottom' if dst == 'neck' else dst)
                    pts.append({'id': [j], 'x': [float(kp[t, 0, s])], 'y': [float(kp[t, 1, s])]})
                hx, hy = kp[t, 0, 2], kp[t, 1, 2]
                rects.append({'x1': [float(hx - 12)], 'y1': [float(hy - 15)], 'x2': [float(hx + 12)], 'y2': [float(hy + 15)],
                              'track_id': [tracks[t]], 'annopoints': [{'point': pts}]})
            annolist.append({'image': [{'name': name}], 'annorect': rects})
        with open(os.path.join(annot, 'vid%03d.json' % v), 'w') as fo:
            json.dump({'annolist': annolist}, fo)
    with open(os.path.join(root, 'roidb.json'), 'w') as fo:
        json.dump(roidb, fo)
    with open(os.path.join(root, 'detections.pkl'), 'wb') as fo:
        pickle.dump({'all_boxes': [[], boxes], 'all_keyps': [[], poses]}, fo)
    return roidb, boxes, poses, annot + os.sep


@pytest.mark.parametrize('command', sorted(README))
def test_compute_tracks_readme_upper_bound_commands(command, tmp_path):
    roidb, boxes, poses, annot = _world(str(tmp_path))
    cfg = tmp_path / 'cfg.yaml'
    cfg.write_text(YAML % (tmp_path / 'roidb.json'))
    out = str(tmp_path / 'out')
    flags = README[command]
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'compute_tracks.py'), '--cfg', str(cfg), 'OUTPUT_DIR', out,
                        'TRACKING.DETECTIONS_FILE', str(tmp_path / 'detections.pkl'), 'EVAL.POSETRACK_ANNOTATION_DIR', annot] + flags,
                       env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    m = re.search(r'\(total mAP, total MOTA\) = \(([^,]+), ([^)]+)\)', r.stdout + r.stderr)
    assert m, r.stdout[-3000:] + r.stderr[-3000:]
    ddir = os.path.join(out, 'test', 'roidb', 'keypoint_rcnn')
    with open(os.path.join(ddir, 'detections_withTracks.pkl'), 'rb') as fi:
        dets = pickle.load(fi)
    # the tracking, against the oracle run on the reference roidb's dtypes (fp32 boxes, int32 keypoints)
    opts = dict(zip(flags[::2], flags[1::2]))
    ub2 = 'TRACKING.DEBUG.UPPER_BOUND_2_GT_KPS' in opts
    ub5 = 'TRACKING.DEBUG.UPPER_BOUND_5_GT_KPS_ONLY' in opts
    for v in range(2):
        idx = [i for i, e in enumerate(roidb) if e['image'].startswith('vid%03d/' % v)]
        frames = [dict(boxes=boxes[i], poses=poses[i], gt_boxes=np.asarray(roidb[i]['boxes'], np.float32),
                       gt_kps=np.asarray(roidb[i]['gt_keypoints']).astype(np.int32), gt_tracks=np.asarray(roidb[i]['tracks']))
                  for i in idx]
        if ub2 or ub5:
            ob, op, ot = U.compute_tracks_video(frames, ub2, ub2, False, ub5)
        else:
            ob, op, ot = [fr['boxes'] for fr in frames], [fr['poses'] for fr in frames], None
        for k, i in enumerate(idx):
            assert np.array_equal(np.asarray(dets['all_boxes'][1][i], np.float32), ob[k]), (v, k)
            assert np.array_equal(np.stack(dets['all_keyps'][1][i]).astype(np.float32), np.stack(op[k]).astype(np.float32)), (v, k)
            if ot is not None and ub2:
                assert dets['all_tracks'][1][i] == ot[k]
    # the score, against the oracle's evaluation of the written files
    json_dir = os.path.join(ddir, 'detections_withTracks.pkl_json') + os.sep
    gt, pr, _ = ope.load_data_dir(annot, json_dir)
    (ap, _, _), metrics, _ = ope.evaluate_frames(gt, pr)
    if 'TRACKING.DEBUG.UPPER_BOUND_4_EVAL_UPPER_BOUND' in opts:
        metrics, _ = U.evaluate_tracking_upper_bound(*ope.load_data_dir(annot, json_dir)[:2])
    got = [float(m.group(1)), float(m.group(2))]
    np.testing.assert_allclose(got, [ap[-1, 0], metrics[-4, 0]], rtol=1e-12, atol=0)
    if ub5:                                                  # GT keypoints on every matched detection
        assert got[0] > 80.0
