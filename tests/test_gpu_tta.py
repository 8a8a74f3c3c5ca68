"""GPU: test-time augmentation (TEST.COMPETITION_MODE) on the device.
  * dt_aug_merge_dets / dt_aug_scale_rois / dt_keypoint_decode_aug bit for bit against numpy restatements (the flip and
    combine of tests/tta_oracle.py, pinned to the reference by tests/golden/tta.npz) and against the unaugmented kernels;
  * the identity plan (COMPETITION_MODE with no extra view) equals COMPETITION_MODE False byte for byte, eager and replayed;
  * end to end against tests/tta_oracle.detect_clip_aug with the criteria of test_gpu_parity_e2e._compare;
  * the batched pipeline equals per-clip im_detect_all with augmentation on."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import tta_oracle as to
from test_gpu_parity_e2e import _match


def _dets(rng, B, C1, R, W, H):
    x1 = rng.uniform(0, W - 1, (B, C1, R)); y1 = rng.uniform(0, H - 1, (B, C1, R))
    d = np.stack([x1, y1, np.minimum(x1 + rng.uniform(0, 90, x1.shape), W - 1), np.minimum(y1 + rng.uniform(0, 90, y1.shape), H - 1),
                  rng.uniform(0.05, 1, x1.shape)], -1)
    return d.astype(np.float32)


@pytest.mark.parametrize('B,C1,R,flips,fill', [(1, 1, 200, (True, False), 'mixed'), (3, 1, 300, (True, False, True, False), 'full'),
                                              (2, 3, 100, (False, True, True), 'zero'), (2, 4, 64, (True,), 'mixed')])
def test_merge_equals_numpy_vstack(B, C1, R, flips, fill):
    import torch
    from detectandtrack_b200.ops import rpn_ops
    rng = np.random.RandomState(B * 7 + C1)
    V = len(flips)
    W = rng.randint(100, 1400, B).astype(np.float32)
    H = 480
    dets = [_dets(rng, B, C1, R, 1400, H) for _ in range(V)]
    if fill == 'full':
        counts = [np.full(B * C1, R, np.int32) for _ in range(V)]
    elif fill == 'zero':
        counts = [np.zeros(B * C1, np.int32)] + [rng.randint(0, R + 1, B * C1).astype(np.int32) for _ in range(V - 1)]
        counts[-1][0] = 0
    else:
        counts = [rng.randint(0, R + 1, B * C1).astype(np.int32) for _ in range(V)]
    im_hw = np.stack([np.full(B, H, np.float32), W], 1)
    out, cnt = rpn_ops.aug_merge_dets([torch.from_numpy(d).cuda() for d in dets], [torch.from_numpy(c).cuda() for c in counts],
                                      flips, torch.from_numpy(im_hw).cuda())
    out, cnt = out.cpu().numpy(), cnt.cpu().numpy()
    for b in range(B):
        for c in range(C1):
            rows = []
            for v in range(V):
                r = dets[v][b, c, :counts[v][b * C1 + c]]
                rows.append(np.hstack([to.flip_boxes(r[:, :4], int(W[b])), r[:, 4:]]) if flips[v] else r)
            ref = np.vstack(rows)
            assert cnt[b * C1 + c] == ref.shape[0]
            assert out[b, c, :ref.shape[0]].tobytes() == ref.tobytes(), (b, c)


def test_scale_rois_aug():
    import torch
    from detectandtrack_b200.ops import dense_ops
    rng = np.random.RandomState(3)
    n, per = 48, 12
    full = _dets(rng, 1, 1, n, 1280, 720)[0, 0]
    boxes = torch.from_numpy(np.hstack([full, np.zeros((n, 3), np.float32)])).cuda()[:, :5]       # row stride 8
    im_hw = torch.tensor([[720., w] for w in (1280., 640., 1000., 333.)], device='cuda')
    scale = 800. / 720.
    a = dense_ops.aug_scale_rois(boxes, scale, False, im_hw, per_image=per)
    b = dense_ops.scale_rois(boxes, 4, scale, per_image=per)
    assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()
    f = dense_ops.aug_scale_rois(boxes, scale, True, im_hw, per_image=per).cpu().numpy()
    widths = im_hw[:, 1].cpu().numpy()
    ref = np.vstack([to.flip_boxes(full[i * per:(i + 1) * per, :4], int(widths[i])) for i in range(n // per)])
    ref = np.hstack([(np.arange(n) // per)[:, None], ref.astype(np.float64) * scale]).astype(np.float32)
    assert f.tobytes() == ref.tobytes()


def _lowres(V, D, K=17, S=14, seed=5):
    import torch
    g = torch.Generator().manual_seed(seed)
    low = torch.randn((V, D, K, 2 * S, 2 * S), generator=g) * 2.0
    low = torch.nn.functional.avg_pool2d(low.view(V * D, K, 2 * S, 2 * S), 3, 1, 1).view(V, D, K, 2 * S, 2 * S) * 3
    ld = 4 * K
    packed = low.view(V, D, K, S, 2, S, 2).permute(0, 1, 3, 5, 4, 6, 2).reshape(V, D, S, S, ld)     # channel (py*2+px)*K + k
    return packed.contiguous().cuda()


def test_keypoint_decode_aug_single_view_is_keypoint_decode():
    import torch
    from detectandtrack_b200.ops import dense_ops
    D = 20
    low = _lowres(1, D)
    boxes = torch.from_numpy(_dets(np.random.RandomState(1), 1, 1, D, 900, 600)[0, 0]).cuda()
    xa, ha = dense_ops.keypoint_decode_aug(low, [False], list(range(17)), False, boxes, 17, want_heatmaps=True)
    xb, hb = dense_ops.keypoint_decode(low[0], boxes, 17, 1, want_heatmaps=True)
    assert xa.cpu().numpy().tobytes() == xb.cpu().numpy().tobytes()
    assert ha.cpu().numpy().tobytes() == hb.cpu().numpy().tobytes()


@pytest.mark.parametrize('hm_max', [False, True])
def test_keypoint_decode_aug_three_views(hm_max):
    import torch
    from detectandtrack_b200.core import tta
    from detectandtrack_b200.ops import dense_ops
    from oracle import keypoints as ok
    D, flips = 16, (False, True, True)
    low = _lowres(3, D, seed=7)
    boxes_np = _dets(np.random.RandomState(2), 1, 1, D, 900, 600)[0, 0]
    boxes = torch.from_numpy(boxes_np).cuda()
    xy, heat = dense_ops.keypoint_decode_aug(low, flips, tta.COCO_FLIP_PERM, hm_max, boxes, 17, want_heatmaps=True)
    views = []
    for v in range(3):
        _, h = dense_ops.keypoint_decode(low[v], boxes, 17, 1, want_heatmaps=True)
        h = h.cpu().numpy()
        views.append(to.flip_heatmaps(h, tta.COCO_FLIP_PERM) if flips[v] else h)
    ref = to.combine(np.stack(views), hm_max)
    heat = heat.cpu().numpy()
    assert heat.tobytes() == np.ascontiguousarray(ref).tobytes()
    got, rxy = xy.cpu().numpy(), ok.heatmaps_to_keypoints(ref, boxes_np, 17)
    np.testing.assert_allclose(got[:, 2], rxy[:, 2], rtol=1e-3, atol=1e-3)
    np.testing.assert_allclose(got[:, 3], rxy[:, 3], rtol=2e-3, atol=1e-6)
    np.testing.assert_allclose(got[:, :2], rxy[:, :2], rtol=0, atol=1e-3)        # the arg-max: peaked maps


def _aug_cfg(**over):
    from test_gpu_engine import _cfg
    cfg = _cfg()
    cfg.TEST.COMPETITION_MODE = True
    cfg.TEST.BBOX_AUG.SCORE_HEUR = 'UNION'; cfg.TEST.BBOX_AUG.COORD_HEUR = 'UNION'
    for k, v in over.items():
        node = cfg
        for p in k.split('.')[:-1]:
            node = node[p]
        node[k.split('.')[-1]] = v
    return cfg


FLIPS = {'TEST.BBOX_AUG.H_FLIP': True, 'TEST.BBOX_AUG.SCALES': (144,), 'TEST.BBOX_AUG.SCALE_H_FLIP': True,
         'TEST.KPS_AUG.H_FLIP': True, 'TEST.KPS_AUG.SCALES': (144,), 'TEST.KPS_AUG.SCALE_H_FLIP': True}


def test_identity_plan_equals_no_augmentation():
    import torch
    from detectandtrack_b200.core import tta
    from detectandtrack_b200.modeling import params as P
    from detectandtrack_b200.modeling.engine import DetectionEngine
    cfg = _aug_cfg()
    blobs, spec = P.random_blobs(cfg, seed=3)
    frames = torch.from_numpy(np.random.RandomState(0).randint(0, 256, (2, 3, 96, 128, 3)).astype(np.uint8)).cuda()
    eng = DetectionEngine(cfg, blobs, spec, dtype='bf16x3')
    plan = tta.view_plan(cfg, spec, 96, 128)
    assert len(plan.box) == len(plan.kps) == 1
    a = eng.detect_static(frames, plan=plan)
    b = eng.detect_static(frames)
    for k in ('dets', 'det_counts', 'xy'):
        assert a[k].cpu().numpy().tobytes() == b[k].cpu().numpy().tobytes(), k
    static_in, run = eng.capture(2, 3, 96, 128, plan=plan)
    static_in.copy_(frames)
    r = run()
    torch.cuda.synchronize()
    for k in ('dets', 'det_counts', 'xy'):
        assert r[k].cpu().numpy().tobytes() == b[k].cpu().numpy().tobytes(), k


def _compare_aug(cfg, blobs, frames, plan, size):
    import torch
    from detectandtrack_b200.modeling import params as P
    from detectandtrack_b200.modeling.engine import DetectionEngine
    ref = to.detect_clip_aug(cfg, blobs, frames, plan)
    eng = DetectionEngine(cfg, blobs, P.GraphSpec(cfg), dtype='bf16x3')
    fr = torch.from_numpy(frames[None]).cuda()
    out = eng.detect_static(fr, want_heatmaps=True, plan=plan)
    res = eng.gather(out)[0]
    b = res['boxes'].cpu().numpy()
    rb = ref['cls_boxes']
    assert b.shape == rb.shape, ('detection count', b.shape, rb.shape)
    assert b.shape[0] > 0
    j, ok = _match(b[:, :4], rb[:, :4], 1e-3 * size)
    assert ok.all() and len(set(j.tolist())) == len(j), ('detections matched', ok.mean())
    assert np.abs(b[:, 4] - rb[j, 4]).max() <= 1e-3, ('scores', np.abs(b[:, 4] - rb[j, 4]).max())
    heat, rheat = res['heatmaps'].cpu().numpy(), ref['heat'][j]
    heat_err = np.abs(heat - rheat).max() / np.abs(rheat).max()
    assert heat_err <= 1e-3, ('combined heat maps', heat_err)
    k, rk = res['keyps'].cpu().numpy(), ref['keyps'][j]
    assert np.abs(k[:, 2] - rk[:, 2]).max() <= 1e-3 * np.abs(rk[:, 2]).max()
    print('tta e2e', dict(n_det=b.shape[0], union=ref['union_count'], heat_err=float(heat_err),
                          box_err=float(np.abs(b[:, :4] - rb[j, :4]).max() / size)))
    return ref


def _union_counts(eng, frames, plan):
    """Rows over the score threshold in the device union (the input of the per-class NMS)."""
    import torch
    from detectandtrack_b200.ops import rpn_ops
    fr = torch.from_numpy(frames[None]).cuda()
    g = eng._geom_tensors(1, frames.shape[1], frames.shape[2])
    d, c = [], []
    for v in plan.box:
        info = eng._view_info(1, v)
        feats = eng._view_features(fr, v)
        rois, _, rc = eng.rpn(feats, info)
        dv, cv_ = eng.box_head_decode(feats, rois, rc, info, g['im_hw'])
        d.append(dv); c.append(cv_)
    _, cnt = rpn_ops.aug_merge_dets(d, c, [v.flip for v in plan.box], g['im_hw'])
    return cnt.cpu().numpy().tolist()


@pytest.mark.parametrize('heur', ['HM_AVG', 'HM_MAX'])
def test_small_clip_matches_oracle(heur):
    from detectandtrack_b200.core import tta
    from detectandtrack_b200.modeling import params as P
    from detectandtrack_b200.modeling.engine import DetectionEngine
    cfg = _aug_cfg(**dict(FLIPS, **{'TEST.KPS_AUG.HEUR': heur}))
    blobs, spec = P.random_blobs(cfg, seed=3)
    frames = np.random.RandomState(0).randint(0, 256, (3, 96, 128, 3)).astype(np.uint8)
    plan = tta.view_plan(cfg, spec, 96, 128)
    assert [v.flip for v in plan.box] == [True, False, True, False] and plan.box[1].size == (144, 192)
    ref = _compare_aug(cfg, blobs, frames, plan, 128.)
    eng = DetectionEngine(cfg, blobs, spec, dtype='bf16x3')
    assert _union_counts(eng, frames, plan) == ref['union_count']


def test_2d_frame_matches_oracle():
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench
    from detectandtrack_b200.core import tta
    from detectandtrack_b200.core.config import reset_cfg
    from detectandtrack_b200.modeling import params as P
    cfg = bench.bench_cfg(256, 320, 'r50fpn2d')
    try:
        cfg.TEST.RPN_POST_NMS_TOP_N = 300
        cfg.TEST.COMPETITION_MODE = True
        cfg.TEST.BBOX_AUG.SCORE_HEUR = 'UNION'; cfg.TEST.BBOX_AUG.COORD_HEUR = 'UNION'
        cfg.TEST.BBOX_AUG.H_FLIP = True; cfg.TEST.KPS_AUG.H_FLIP = True
        blobs, spec = P.random_blobs(cfg, seed=11)
        frames = np.random.RandomState(2).randint(0, 256, (1, 256, 320, 3)).astype(np.uint8)
        _compare_aug(cfg, blobs, frames, tta.view_plan(cfg, spec, 256, 320), 320.)
    finally:
        reset_cfg()


def test_batched_pipeline_equals_per_clip():
    from detectandtrack_b200.core.test import im_detect_all, im_detect_all_batch
    from detectandtrack_b200.modeling import params as P
    from detectandtrack_b200.modeling import model_builder
    cfg = _aug_cfg(**FLIPS)
    blobs, _ = P.random_blobs(cfg, seed=3)
    model = model_builder.create(cfg.MODEL.TYPE, train=False, blobs=blobs)
    rng = np.random.RandomState(4)
    ims = [[rng.randint(0, 256, (96, 128, 3)).astype(np.uint8) for _ in range(3)] for _ in range(4)]
    batched = im_detect_all_batch(model, ims, clips_per_step=4)
    for im, (bb, _, bk) in zip(ims, batched):
        rb, _, rk = im_detect_all(model, im)
        assert bb[1].tobytes() == rb[1].tobytes()
        assert (bk is None) == (rk is None)
        if bk is not None:
            assert np.stack(bk[1]).tobytes() == np.stack(rk[1]).tobytes()


def test_test_net_competition_mode_then_compute_tracks(tmp_path):
    """tools/test_net.py with TEST.COMPETITION_MODE and box / keypoint H_FLIP writes a detections.pkl of the usual schema,
    which tools/compute_tracks.py reads."""
    import pickle
    import subprocess
    from test_gpu_tools import YAML, ROOT
    aug = ('COMPETITION_MODE: True\n  BBOX_AUG:\n    SCORE_HEUR: UNION\n    COORD_HEUR: UNION\n    H_FLIP: True\n'
           '  KPS_AUG:\n    H_FLIP: True\n')
    assert 'COMPETITION_MODE: False\n' in YAML
    cfg = tmp_path / 'cfg.yaml'
    cfg.write_text(YAML.replace('COMPETITION_MODE: False\n', aug))
    out = str(tmp_path / 'out')
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'test_net.py'), '--cfg', str(cfg), 'OUTPUT_DIR', out],
                       env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    ddir = os.path.join(out, 'test', 'synthetic_2x3_96x128', 'keypoint_rcnn')
    det = pickle.load(open(os.path.join(ddir, 'detections.pkl'), 'rb'))
    assert 'COMPETITION_MODE: true' in det['cfg'] and len(det['all_boxes'][1]) == 6
    assert sum(b.shape[0] for b in det['all_boxes'][1]) > 0
    for i in range(6):
        b = det['all_boxes'][1][i]
        assert b.dtype == np.float32 and b.shape[1] == 5 and len(det['all_keyps'][1][i]) == b.shape[0]
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'compute_tracks.py'), '--cfg', str(cfg), 'OUTPUT_DIR', out],
                       env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    trk = pickle.load(open(os.path.join(ddir, 'detections_withTracks.pkl'), 'rb'))
    assert len(trk['all_tracks'][1]) == 6
    assert [len(t) for t in trk['all_tracks'][1]] == [b.shape[0] for b in trk['all_boxes'][1]]     # confidence-filtered boxes
