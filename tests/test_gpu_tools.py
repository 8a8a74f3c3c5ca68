"""GPU: the reference's two entry points end to end on a synthetic dataset:
tools/test_net.py (detections.pkl schema) -> tools/compute_tracks.py (detections_withTracks.pkl)."""
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

YAML = '''
MODEL:
  TYPE: keypoint_rcnn
  CONV_BODY: FPN3D.add_fpn_ResNet50_conv5_body
  ROI_HEAD: head_builder.add_roi_2mlp_head
  NUM_CLASSES: 2
  FASTER_RCNN: True
  KEYPOINTS_ON: True
  VIDEO_ON: True
FPN:
  FPN_ON: True
  MULTILEVEL_ROIS: True
  MULTILEVEL_RPN: True
FAST_RCNN:
  ROI_XFORM_METHOD: RoIAlign
  ROI_XFORM_RESOLUTION: 7
  ROI_XFORM_SAMPLING_RATIO: 2
KRCNN:
  ROI_KEYPOINTS_HEAD: keypoint_rcnn_heads.add_roi_pose_head_v1convX
  NUM_STACKED_CONVS: 8
  NUM_KEYPOINTS: 17
  USE_DECONV_OUTPUT: True
  CONV_HEAD_DIM: 512
  UP_SCALE: 2
  HEATMAP_SIZE: 56
  ROI_XFORM_RESOLUTION: 14
  ROI_XFORM_SAMPLING_RATIO: 2
VIDEO:
  NUM_FRAMES: 3
  TIME_INTERVAL: 1
  WEIGHTS_INFLATE_MODE: center-only
  TIME_KERNEL_DIM: 3
  BODY_HEAD_LINK: 'slice-center'
  NUM_FRAMES_MID: 1
TEST:
  DATASET: synthetic_2x3_96x128
  WEIGHTS: random
  SCALES: (96,)
  MAX_SIZE: 128
  NMS: 0.5
  RPN_PRE_NMS_TOP_N: 1000
  RPN_POST_NMS_TOP_N: 300
  COMPETITION_MODE: False
TRACKING:
  CONF_FILTER_INITIAL_DETS: 0.3
  DISTANCE_METRICS: ('bbox-overlap', 'cnn-cosdist')
  DISTANCE_METRIC_WTS: (1.0, 0.0)
  BIPARTITE_MATCHING_ALGO: 'hungarian'
NUM_GPUS: 1
'''


def test_test_net_then_compute_tracks(tmp_path):
    cfg = tmp_path / 'cfg.yaml'
    cfg.write_text(YAML)
    out = str(tmp_path / 'out')
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'test_net.py'), '--cfg', str(cfg), 'OUTPUT_DIR', out],
                       env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    ddir = os.path.join(out, 'test', 'synthetic_2x3_96x128', 'keypoint_rcnn')
    det = pickle.load(open(os.path.join(ddir, 'detections.pkl'), 'rb'))
    assert set(det) >= {'all_boxes', 'all_segms', 'all_keyps', 'cfg'}
    assert len(det['all_boxes']) == 2 and len(det['all_boxes'][1]) == 6
    for i in range(6):
        b = det['all_boxes'][1][i]
        assert b.dtype == np.float32 and b.ndim == 2 and b.shape[1] == 5
        assert len(det['all_keyps'][1][i]) == b.shape[0]
        if b.shape[0]:
            assert det['all_keyps'][1][i][0].shape == (4, 17)
    # test_net on a posetrack-like dataset runs tracking itself (test_engine.py:326-328)
    trk = pickle.load(open(os.path.join(ddir, 'detections_withTracks.pkl'), 'rb'))
    assert len(trk['all_tracks'][1]) == 6
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'compute_tracks.py'), '--cfg', str(cfg), 'OUTPUT_DIR', out],
                       env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    trk2 = pickle.load(open(os.path.join(ddir, 'detections_withTracks.pkl'), 'rb'))
    assert trk2['all_tracks'][1] == trk['all_tracks'][1]
    for i in range(6):
        assert len(trk2['all_tracks'][1][i]) == trk2['all_boxes'][1][i].shape[0]
    # ids restart per video (2 videos x 3 frames): first frame of each video starts at FIRST_TRACK_ID
    for first in (0, 3):
        ids = trk2['all_tracks'][1][first]
        assert ids == list(range(len(ids)))


TRAIN_YAML = YAML + '''
TRAIN:
  DATASET: synthetic_1x2_96x128
  SCALES: (96,)
  MAX_SIZE: 128
  IMS_PER_BATCH: 2
  BATCH_SIZE_PER_IM: 64
  RPN_BATCH_SIZE_PER_IM: 64
  RPN_PRE_NMS_TOP_N: 300
  RPN_POST_NMS_TOP_N: 200
SOLVER:
  BASE_LR: 0.0003
  LR_POLICY: steps_with_decay
  STEPS: [0, 30]
  MAX_ITER: 61
  WARM_UP_ITERS: 5
  WEIGHT_DECAY: 0.0001
'''


def test_train_net_loss_goes_down(tmp_path):
    """tools/train_net.py (reference CLI) on a 2-clip synthetic dataset: the same minibatch every iteration, so the total loss
    of the keypoint R-CNN step must fall (lr 3e-4 with warm-up and one decay step)."""
    import re
    cfg = tmp_path / 'cfg.yaml'
    cfg.write_text(TRAIN_YAML)
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'train_net.py'), '--cfg', str(cfg), 'OUTPUT_DIR', str(tmp_path / 'out')],
                       env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    losses = [float(m.group(1)) for m in re.finditer(r'iter \d+ lr [\d.]+ loss ([\d.]+)', r.stdout)]
    assert len(losses) == 4 and all(np.isfinite(losses)), r.stdout[-2000:]
    # the snapshot is a weights file of the reference's format that tools/test_net.py runs on
    snap = os.path.join(str(tmp_path / 'out'), 'train', 'synthetic_1x2_96x128', 'keypoint_rcnn', 'model_final.pkl')
    w = pickle.load(open(snap, 'rb'))
    assert 'blobs' in w and w['blobs']['fc6_w'].shape == (1024, 12544) and w['blobs']['kps_score_lowres_w'].shape == (512, 17, 4, 4)
    r2 = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'test_net.py'), '--cfg', str(cfg), 'OUTPUT_DIR', str(tmp_path / 'out2'),
                         'TEST.WEIGHTS', snap], env=env, capture_output=True, text=True, timeout=600)
    assert r2.returncode == 0, r2.stdout[-2000:] + r2.stderr[-2000:]
    assert os.path.exists(os.path.join(str(tmp_path / 'out2'), 'test', 'synthetic_2x3_96x128', 'keypoint_rcnn', 'detections.pkl'))
    assert losses[-1] < 0.7 * losses[0], losses          # lr 3e-4, new RoI draws every iteration (1e-3 sits at the edge
                                                         # of stability of these random weights, 2e-3 diverges)


def test_multi_gpu_testing_equals_single_gpu(tmp_path):
    """tools/test_net.py --multi-gpu-testing (lib/utils/subprocess.py:27-74: one child per GPU over contiguous index ranges,
    results concatenated in rank order, no collective) gives the detections of the single-process run, bit for bit."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    cfg = tmp_path / 'cfg.yaml'
    cfg.write_text(YAML)
    env = dict(os.environ, PYTHONPATH=ROOT)
    outs = []
    for tag, extra in (('one', []), ('two', ['--multi-gpu-testing'])):
        out = str(tmp_path / tag)
        r = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'test_net.py'), '--cfg', str(cfg)] + extra +
                           ['OUTPUT_DIR', out, 'NUM_GPUS', '2' if extra else '1'], env=env, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        outs.append(pickle.load(open(os.path.join(out, 'test', 'synthetic_2x3_96x128', 'keypoint_rcnn', 'detections.pkl'), 'rb')))
    a, b = outs
    assert len(a['all_boxes'][1]) == len(b['all_boxes'][1]) == 6
    for i in range(6):
        assert np.array_equal(a['all_boxes'][1][i], b['all_boxes'][1][i])
        assert len(a['all_keyps'][1][i]) == len(b['all_keyps'][1][i])
        for ka, kb in zip(a['all_keyps'][1][i], b['all_keyps'][1][i]):
            assert np.array_equal(ka, kb)
