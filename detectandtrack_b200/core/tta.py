"""Test-time augmentation plan (TEST.COMPETITION_MODE; lib/core/test.py:255-414, 630-747, 897-958).

The cfg maps to two ordered view lists, in the reference's order:
  box stage (im_detect_bbox_aug):      H_FLIP; per BBOX_AUG.SCALES s: s, then its flip if SCALE_H_FLIP; identity last
  keypoint stage (im_detect_keypoints_aug): identity first; H_FLIP; per KPS_AUG.SCALES s: s, then its flip if SCALE_H_FLIP
Each view is (flip, im_scale, resized (hr, wr), padded (hp, wp)) for an H x W clip.  A scale view runs with
TEST.SCALES = (s,) and TEST.MAX_SIZE = that stage's MAX_SIZE; the identity and H_FLIP views with TEST.SCALES[0] and
TEST.MAX_SIZE.  Every check of what the device path can run lives here (view_plan), before anything is built."""
import collections

from ..modeling.engine import check_box_post, im_scale_and_size, padded_blob_size

View = collections.namedtuple('View', 'flip im_scale size padded')
Plan = collections.namedtuple('Plan', 'box kps hm_max perm')

# flip_heatmaps swaps left and right joints by the COCO map of get_keypoints (lib/utils/keypoints.py:28-58, 81-91),
# whatever the dataset: joint k of a flipped view's combined map is joint COCO_FLIP_PERM[k] of its own map.
COCO_FLIP_PERM = (0, 2, 1, 4, 3, 6, 5, 8, 7, 10, 9, 12, 11, 14, 13, 16, 15)

MAX_VIEWS = 16                  # DT_AUG_MAX_VIEWS: views per stage
NMS_MAX_BOXES = 8192            # DT_NMS_MAX_BOXES: per (image, class) union
LIMIT_MAX_ROWS = 16384          # dt_limit_detections: (C-1) x union rows per image


def _check(cfg, spec):
    box, kps = cfg.TEST.BBOX_AUG, cfg.TEST.KPS_AUG
    # the reference's own assertions (lib/core/test.py:338-346, 721-722), with its messages
    assert not box.SCALE_SIZE_DEP, 'Size dependent scaling not implemented'
    assert not box.SCORE_HEUR == 'UNION' or box.COORD_HEUR == 'UNION', \
        'Coord heuristic must be union whenever score heuristic is union'
    assert not box.COORD_HEUR == 'UNION' or box.SCORE_HEUR == 'UNION', \
        'Score heuristic must be union whenever coord heuristic is union'
    assert not cfg.MODEL.FASTER_RCNN or box.SCORE_HEUR == 'UNION', \
        'Union heuristic must be used to combine Faster RCNN predictions'
    if box.SCORE_HEUR != 'UNION':
        raise NotImplementedError('test-time augmentation: box heuristics %s / %s need precomputed proposals, which are '
                                  'not on the hot path' % (box.SCORE_HEUR, box.COORD_HEUR))
    if cfg.MODEL.KEYPOINTS_ON:
        assert not kps.SCALE_SIZE_DEP, 'Size dependent scaling not implemented'
        if kps.HEUR not in ('HM_AVG', 'HM_MAX'):
            raise NotImplementedError('Heuristic {} not supported'.format(kps.HEUR))
        if kps.ASPECT_RATIOS:
            raise NotImplementedError('test-time augmentation: KPS_AUG.ASPECT_RATIOS (the reference resamples the frames '
                                      'to uint8 before the blob resize) is not on the hot path')
    if box.ASPECT_RATIOS:
        raise NotImplementedError('test-time augmentation: BBOX_AUG.ASPECT_RATIOS (the reference resamples the frames '
                                  'to uint8 before the blob resize) is not on the hot path')
    if spec is not None and (not spec.fpn or spec.head3d):
        raise NotImplementedError('test-time augmentation: FPN graphs with 2-D heads only (not tube heads)')
    check_box_post(cfg, spec)


def _stage(cfg, aug, identity_first, H, W, stride):
    base = (cfg.TEST.SCALES[0], cfg.TEST.MAX_SIZE)
    keys = [(False,) + base] if identity_first else []
    if aug.H_FLIP:
        keys.append((True,) + base)
    for s in aug.SCALES:
        keys.append((False, s, aug.MAX_SIZE))
        if aug.SCALE_H_FLIP:
            keys.append((True, s, aug.MAX_SIZE))
    if not identity_first:
        keys.append((False,) + base)
    views = []
    for flip, target, max_size in keys:
        scale, size = im_scale_and_size(H, W, target, max_size)
        views.append(View(flip, scale, size, padded_blob_size([size], stride)))
    return tuple(views)


def view_plan(cfg, spec, H, W):
    """The TEST.COMPETITION_MODE plan of an H x W clip for the graph `spec` (None: skip the graph check).
    Raises, before any device work, for what the reference rejects and for what the device path does not run."""
    _check(cfg, spec)
    stride = int(cfg.FPN.COARSEST_STRIDE) if cfg.FPN.FPN_ON else 1
    box = _stage(cfg, cfg.TEST.BBOX_AUG, False, H, W, stride)
    kps = _stage(cfg, cfg.TEST.KPS_AUG, True, H, W, stride) if cfg.MODEL.KEYPOINTS_ON else ()
    post = cfg.TEST.RPN_POST_NMS_TOP_N
    R = post if post > 0 else (cfg.FPN.RPN_MAX_LEVEL - cfg.FPN.RPN_MIN_LEVEL + 1) * cfg.TEST.RPN_PRE_NMS_TOP_N   # collect's R
    V, C1 = len(box), cfg.MODEL.NUM_CLASSES - 1
    if max(V, len(kps)) > MAX_VIEWS:
        raise ValueError('test-time augmentation: %d box / %d keypoint views exceed %d' % (V, len(kps), MAX_VIEWS))
    if V * R > NMS_MAX_BOXES:
        raise ValueError('test-time augmentation: %d box views x %d proposals = %d union rows per class exceed the NMS '
                         'capacity of %d' % (V, R, V * R, NMS_MAX_BOXES))
    if C1 * V * R > LIMIT_MAX_ROWS:
        raise ValueError('test-time augmentation: %d classes x %d box views x %d proposals = %d union rows per image exceed '
                         'the DETECTIONS_PER_IM limit capacity of %d' % (C1, V, R, C1 * V * R, LIMIT_MAX_ROWS))
    K = cfg.KRCNN.NUM_KEYPOINTS
    perm = tuple(range(K))
    if any(v.flip for v in kps):
        if K != len(COCO_FLIP_PERM):
            raise NotImplementedError('test-time augmentation: flip_heatmaps swaps the %d COCO joints; this model has %d'
                                      % (len(COCO_FLIP_PERM), K))
        perm = COCO_FLIP_PERM
    return Plan(box, kps, cfg.TEST.KPS_AUG.HEUR == 'HM_MAX', perm)
