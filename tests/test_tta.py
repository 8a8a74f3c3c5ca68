"""CPU: the test-time augmentation plan (core/tta.py) — view order and geometry, every rejection before device work —
the TTA oracle's flip and combine pinned bit for bit to the reference's own functions (tests/golden/tta.npz), and the
new C entry points rejecting bad arguments on the host before any CUDA call."""
import ctypes as C
import os

import numpy as np
import pytest

from detectandtrack_b200 import _lib as L

HERE = os.path.dirname(os.path.abspath(__file__))


def _cfg(**over):
    from detectandtrack_b200.core.config import cfg, reset_cfg, assert_and_infer_cfg
    reset_cfg()
    cfg.MODEL.TYPE = 'keypoint_rcnn'
    cfg.MODEL.CONV_BODY = 'FPN3D.add_fpn_ResNet50_conv5_body'
    cfg.MODEL.NUM_CLASSES = 2
    cfg.MODEL.FASTER_RCNN = True
    cfg.MODEL.KEYPOINTS_ON = True
    cfg.KRCNN.NUM_KEYPOINTS = 17
    cfg.FPN.FPN_ON = True
    cfg.TEST.SCALES = (800,); cfg.TEST.MAX_SIZE = 1333
    cfg.TEST.RPN_POST_NMS_TOP_N = 1000
    cfg.TEST.COMPETITION_MODE = True
    cfg.TEST.BBOX_AUG.SCORE_HEUR = 'UNION'; cfg.TEST.BBOX_AUG.COORD_HEUR = 'UNION'
    for k, v in over.items():
        node = cfg
        parts = k.split('.')
        for p in parts[:-1]:
            node = node[p]
        node[parts[-1]] = v
    return cfg


def _plan(H=720, W=1280, **over):
    from detectandtrack_b200.core import tta
    return tta.view_plan(_cfg(**over), None, H, W)


def _key(v):
    return (v.flip, round(v.im_scale, 12), v.size, v.padded)


def test_identity_plan():
    p = _plan()
    assert [_key(v) for v in p.box] == [(False, round(1333 / 1280., 12), (750, 1333), (768, 1344))]     # MAX_SIZE binds
    assert p.kps == p.box and not p.hm_max and p.perm == tuple(range(17))


def test_view_order_and_geometry():
    from detectandtrack_b200.modeling.engine import im_scale_and_size, padded_blob_size
    p = _plan(**{'TEST.BBOX_AUG.H_FLIP': True, 'TEST.BBOX_AUG.SCALES': (400, 1200), 'TEST.BBOX_AUG.SCALE_H_FLIP': True,
                 'TEST.BBOX_AUG.MAX_SIZE': 2000, 'TEST.KPS_AUG.H_FLIP': True, 'TEST.KPS_AUG.SCALES': (600,),
                 'TEST.KPS_AUG.SCALE_H_FLIP': True, 'TEST.KPS_AUG.MAX_SIZE': 900, 'TEST.KPS_AUG.HEUR': 'HM_MAX'})

    def geo(flip, target, max_size):
        sc, size = im_scale_and_size(720, 1280, target, max_size)
        return (flip, round(sc, 12), size, padded_blob_size([size], 32))
    base = (800, 1333)
    assert [_key(v) for v in p.box] == [geo(True, *base), geo(False, 400, 2000), geo(True, 400, 2000), geo(False, 1200, 2000),
                                        geo(True, 1200, 2000), geo(False, *base)]
    assert [_key(v) for v in p.kps] == [geo(False, *base), geo(True, *base), geo(False, 600, 900), geo(True, 600, 900)]
    assert p.box[3].size == (1125, 2000)                       # MAX_SIZE caps the long side
    assert p.kps[2].size == (506, 900)
    assert p.hm_max and p.perm == (0, 2, 1, 4, 3, 6, 5, 8, 7, 10, 9, 12, 11, 14, 13, 16, 15)


def test_scales_without_scale_flip_and_no_keypoints():
    p = _plan(**{'TEST.BBOX_AUG.SCALES': (500,), 'TEST.KPS_AUG.H_FLIP': True, 'MODEL.KEYPOINTS_ON': False})
    assert [v.flip for v in p.box] == [False, False] and p.box[0].size == (500, 889) and p.kps == ()


@pytest.mark.parametrize('over,exc,msg', [
    ({'TEST.BBOX_AUG.SCALE_SIZE_DEP': True}, AssertionError, 'Size dependent scaling not implemented'),
    ({'TEST.KPS_AUG.SCALE_SIZE_DEP': True}, AssertionError, 'Size dependent scaling not implemented'),
    ({'TEST.BBOX_AUG.SCORE_HEUR': 'ID', 'TEST.BBOX_AUG.COORD_HEUR': 'ID'}, AssertionError,
     'Union heuristic must be used to combine Faster RCNN predictions'),
    ({'TEST.BBOX_AUG.SCORE_HEUR': 'AVG', 'TEST.BBOX_AUG.COORD_HEUR': 'AVG'}, AssertionError,
     'Union heuristic must be used to combine Faster RCNN predictions'),
    ({'TEST.BBOX_AUG.COORD_HEUR': 'ID'}, AssertionError, 'Coord heuristic must be union whenever score heuristic is union'),
    ({'TEST.BBOX_AUG.SCORE_HEUR': 'AVG'}, AssertionError, 'Score heuristic must be union whenever coord heuristic is union'),
    ({'TEST.KPS_AUG.HEUR': 'HM_MEDIAN'}, NotImplementedError, 'Heuristic HM_MEDIAN not supported'),
    ({'TEST.BBOX_AUG.ASPECT_RATIOS': (0.5,)}, NotImplementedError, 'BBOX_AUG.ASPECT_RATIOS'),
    ({'TEST.KPS_AUG.ASPECT_RATIOS': (2.0,)}, NotImplementedError, 'KPS_AUG.ASPECT_RATIOS'),
    ({'TEST.BBOX_AUG.H_FLIP': True, 'TEST.BBOX_AUG.SCALES': (400, 500, 600, 700), 'TEST.BBOX_AUG.SCALE_H_FLIP': True},
     ValueError, 'exceed the NMS capacity of 8192'),
    ({'TEST.BBOX_AUG.SCALES': (400, 500), 'MODEL.NUM_CLASSES': 7}, ValueError, 'limit capacity of 16384'),
    ({'TEST.KPS_AUG.H_FLIP': True, 'KRCNN.NUM_KEYPOINTS': 15}, NotImplementedError, 'swaps the 17 COCO joints'),
])
def test_rejections(over, exc, msg):
    with pytest.raises(exc, match=msg):
        _plan(**over)


def test_tube_heads_rejected():
    from detectandtrack_b200.core import tta

    class Spec(object):
        fpn, head3d = False, True
    with pytest.raises(NotImplementedError, match='not tube heads'):
        tta.view_plan(_cfg(), Spec(), 720, 1280)


def test_default_competition_mode_is_the_reference_assertion():
    """COMPETITION_MODE defaults to True with the ID heuristics, which the reference rejects for Faster R-CNN models."""
    from detectandtrack_b200.core import tta
    cfg = _cfg(**{'TEST.BBOX_AUG.SCORE_HEUR': 'ID', 'TEST.BBOX_AUG.COORD_HEUR': 'ID'})
    with pytest.raises(AssertionError, match='Union heuristic'):
        tta.view_plan(cfg, None, 96, 128)


def test_oracle_flip_and_combine_match_the_reference():
    import tta_oracle as to
    from detectandtrack_b200.core import tta
    g = np.load(os.path.join(HERE, 'golden', 'tta.npz'))
    got = to.flip_boxes(g['boxes'], int(g['width']))
    assert got.dtype == np.float32 and got.tobytes() == g['boxes_flipped'].tobytes()
    f1 = to.flip_heatmaps(g['maps'][1], tta.COCO_FLIP_PERM)
    assert np.ascontiguousarray(f1).tobytes() == g['maps_flip1'].tobytes()
    views = np.stack([g['maps'][0], f1, g['maps'][2]])
    for hm_max, key in ((False, 'hm_avg'), (True, 'hm_max')):
        c = to.combine(views, hm_max)
        assert c.dtype == np.float32 and c.tobytes() == g[key].tobytes(), key


def _aug_cases():
    P = lambda n: (C.c_void_p * n)(*([None] * n))
    I = lambda *v: (C.c_int * len(v))(*v)
    perm = I(*range(17))
    bad_perm = I(*([0] * 17))
    return [
        ('dt_aug_merge_dets', (P(2), P(2), I(0, 1), 0, 1, 2, 1000, None, 2, None, None, None), b'V=0'),
        ('dt_aug_merge_dets', (P(17), P(17), I(*[0] * 17), 17, 1, 2, 100, None, 2, None, None, None), b'V=17'),
        ('dt_aug_merge_dets', (P(2), P(2), I(0, 1), 2, 1, 1, 1000, None, 2, None, None, None), b'bad shape'),
        ('dt_aug_merge_dets', (P(9), P(9), I(*[0] * 9), 9, 1, 2, 1000, None, 2, None, None, None), b'V*R=9000 exceeds 8192'),
        ('dt_aug_merge_dets', (P(2), P(2), I(0, 1), 2, 1, 2, 1000, None, 2, None, None, None), b'view 0 null pointer'),
        ('dt_aug_scale_rois', (None, 3, 10, 0, None, 2, 1, 1.0, None, None), b'bad shape'),
        ('dt_aug_scale_rois', (None, 5, 10, 1, None, 2, 1, 1.0, None, None), b'null pointer'),
        ('dt_keypoint_decode_aug', (None, 0, 68, 99, 17, 1, I(0), perm, 0, None, 4, None, 10, 0, None, None, None), b'S=99'),
        ('dt_keypoint_decode_aug', (None, 10 * 14 * 14 * 68, 68, 14, 17, 0, I(0), perm, 0, None, 4, None, 10, 0, None, None, None),
         b'V=0'),
        ('dt_keypoint_decode_aug', (None, 100, 68, 14, 17, 2, I(0, 1), perm, 0, None, 4, None, 10, 0, None, None, None),
         b'view_stride'),
        ('dt_keypoint_decode_aug', (None, 10 * 14 * 14 * 68, 68, 14, 17, 2, I(0, 1), perm, 2, None, 4, None, 10, 0, None, None, None),
         b'hm_max'),
        ('dt_keypoint_decode_aug', (None, 10 * 14 * 14 * 68, 68, 14, 17, 2, I(0, 1), bad_perm, 0, None, 4, None, 10, 0, None, None,
                                    None), b'not a permutation'),
        ('dt_keypoint_decode_aug', (None, 10 * 14 * 14 * 68, 68, 14, 17, 2, I(0, 1), perm, 0, None, 4, None, 10, 0, None, None, None),
         b'null pointer'),
    ]


@pytest.mark.parametrize('name,args,msg', _aug_cases(), ids=['%s-%d' % (c[0], i) for i, c in enumerate(_aug_cases())])
def test_aug_entry_points_reject_bad_arguments_without_a_gpu(name, args, msg):
    lib = L.lib()
    rc = getattr(lib, name)(*args)
    err = lib.dt_last_error()
    assert rc != 0, name
    assert msg in err, (name, err)
    with pytest.raises(RuntimeError, match=name):
        L.check(rc, name)
