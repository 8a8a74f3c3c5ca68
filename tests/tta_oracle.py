"""Oracle of the test-time augmented inference path (TEST INFRASTRUCTURE ONLY): ONE clip through the reference's
COMPETITION_MODE flow on the CPU in fp32, composed from the oracle package's per-stage restatements:

  lib/core/test.py:897-958 (im_detect_all), :255-414 (im_detect_bbox_aug, UNION / UNION), :630-747
  (im_detect_keypoints_aug), lib/utils/blob.py:71-90 (prep_im_for_blob), lib/utils/boxes.py:275-282 (flip_boxes),
  lib/utils/keypoints.py:81-91 (flip_heatmaps)

Each view's blob is cv2 INTER_LINEAR on the mean-subtracted frames, mirrored first where the view flips.  A box view
decodes all R proposals in original-image coordinates and a flipped one is flipped back class slice by class slice
(the reference's flip_boxes asserts 4 columns; DESIGN.md §4); the views' rows are stacked in view order and go through
box_results_with_nms_and_limit.  The keypoint views run on the final boxes; flipped maps go through flip_heatmaps, the
maps are combined with np.mean / np.amax over the views and keypoint_results decodes them against the final boxes.
The flip and combine restatements below are pinned to the reference's own functions by tests/golden/tta.npz."""
import numpy as np

from oracle import net as onet, proposals as oprop, detections as odet, keypoints as okp
from oracle.graph import OracleSpec

F32 = np.float32


def flip_boxes(boxes, im_width):
    """flip_boxes on every 4-column slice of boxes [n, 4k] (fp32; numpy's `im_width - x - 1`)."""
    out = boxes.copy()
    out[:, 0::4] = im_width - boxes[:, 2::4] - 1
    out[:, 2::4] = im_width - boxes[:, 0::4] - 1
    return out


def flip_heatmaps(heatmaps, perm):
    """flip_heatmaps: joint k of the result is joint perm[k] of the input, mirrored in x."""
    return heatmaps[:, list(perm)][:, :, :, ::-1]


def combine(maps, hm_max):
    """HM_MAX: np.amax over the views; HM_AVG: np.mean."""
    return np.amax(maps, axis=0) if hm_max else np.mean(maps, axis=0)


def view_blob(cfg, frames, view):
    """frames [T, H, W, 3] uint8 -> the view's blob [T, hp, wp, 3] fp32 (prep_im_for_blob + im_list_to_blob)."""
    import cv2
    T = frames.shape[0]
    (hr, wr), (hp, wp) = view.size, view.padded
    means = np.asarray(cfg.PIXEL_MEANS, F32).reshape(1, 1, 3)
    blob = np.zeros((T, hp, wp, 3), F32)
    for t in range(T):
        im = frames[t][:, ::-1] if view.flip else frames[t]
        im = im.astype(F32) - means
        im = cv2.resize(im, None, None, fx=view.im_scale, fy=view.im_scale, interpolation=cv2.INTER_LINEAR)
        assert im.shape[:2] == (hr, wr), (im.shape, view)
        blob[t, :hr, :wr] = im
    return blob


def _features(cfg, blobs, spec, blob):
    import torch
    if spec.is3d:
        data = torch.from_numpy(blob)[None].permute(0, 4, 1, 2, 3).contiguous()
    else:
        data = torch.from_numpy(blob).permute(0, 3, 1, 2).contiguous()
    pyr = onet.fpn(blobs, spec, onet.conv_body(blobs, spec, data))
    return [onet.time_pool(p, spec.link, cfg.VIDEO.NUM_FRAMES_MID) for p in pyr][::-1]       # P2..P6


def detect_clip_aug(cfg, blobs, frames, plan, spec=None):
    """frames [T, H, W, 3] uint8 BGR; plan = core/tta.view_plan(cfg, ...) of this H x W.  Returns dict(cls_boxes [n, 5],
    keyps [n, 4, K], heat (n, K, 56, 56) combined maps, union_count = rows over the score threshold in the union)."""
    import torch
    npy = lambda t: t.detach().float().cpu().numpy()
    spec = spec or OracleSpec(cfg)
    assert spec.fpn and not spec.head3d, 'oracle: FPN graphs with 2-D heads'
    H, W = frames.shape[1:3]
    R, D = cfg.TEST.RPN_POST_NMS_TOP_N, cfg.TEST.DETECTIONS_PER_IM
    C, K = cfg.MODEL.NUM_CLASSES, cfg.KRCNN.NUM_KEYPOINTS
    nl = len(spec.roi_levels)
    scales = [1. / 2 ** l for l in spec.roi_levels]
    scores_ts, boxes_ts = [], []
    with torch.no_grad():
        for v in plan.box:
            feats = _features(cfg, blobs, spec, view_blob(cfg, frames, v))
            im_info = np.array([v.padded[0], v.padded[1], v.im_scale], F32)
            rois_l, sc_l = [], []
            for l, (lg, dl) in enumerate(onet.rpn_heads_fpn(blobs, spec, feats[::-1])):
                lvl = spec.rpn_levels[l]
                anchors = oprop.generate_anchors(2. ** lvl, (cfg.FPN.RPN_ANCHOR_START_SIZE * 2. ** (lvl - spec.rpn_levels[0]),),
                                                 cfg.FPN.RPN_ASPECT_RATIOS)
                p, s = oprop.generate_proposals(npy(torch.sigmoid(lg.float())[0]), npy(dl[0]), im_info, anchors, 2. ** lvl,
                                                cfg.TEST.RPN_PRE_NMS_TOP_N, cfg.TEST.RPN_POST_NMS_TOP_N,
                                                cfg.TEST.RPN_NMS_THRESH, cfg.TEST.RPN_MIN_SIZE)
                rois_l.append(np.hstack([np.zeros((p.shape[0], 1), F32), p])); sc_l.append(s)
            rois = oprop.collect(rois_l, sc_l, R)
            cls, bbox = onet.box_head_2mlp(blobs, onet.roi_features(feats[:nl], scales, rois, cfg.FAST_RCNN.ROI_XFORM_RESOLUTION,
                                                                    cfg.FAST_RCNN.ROI_XFORM_SAMPLING_RATIO,
                                                                    spec.roi_levels[0], spec.roi_levels[-1]))
            boxes = odet.decode_boxes(rois, npy(bbox), v.im_scale, (H, W), cfg.MODEL.BBOX_REG_WEIGHTS)
            scores_ts.append(odet.softmax(npy(cls)))
            boxes_ts.append(flip_boxes(boxes, W) if v.flip else boxes)
        scores_c, boxes_c = np.vstack(scores_ts), np.vstack(boxes_ts)
        union_count = [int((scores_c[:, j] > F32(cfg.TEST.SCORE_THRESH)).sum()) for j in range(1, C)]
        _, det_boxes, cls_boxes = odet.box_results_with_nms_and_limit(scores_c, boxes_c, C, cfg.TEST.SCORE_THRESH,
                                                                      cfg.TEST.NMS, D)
        keyps, heat = None, None
        if cfg.MODEL.KEYPOINTS_ON and det_boxes.shape[0]:
            maps = []
            for v in plan.kps:
                feats = _features(cfg, blobs, spec, view_blob(cfg, frames, v))
                b = flip_boxes(det_boxes[:, :4], W) if v.flip else det_boxes[:, :4]
                kr = np.hstack([np.zeros((b.shape[0], 1)), b.astype(np.float64) * v.im_scale]).astype(F32)   # _get_rois_blob
                h, _ = onet.keypoint_head_2d(blobs, onet.roi_features(feats[:nl], scales, kr, cfg.KRCNN.ROI_XFORM_RESOLUTION,
                                                                      cfg.KRCNN.ROI_XFORM_SAMPLING_RATIO,
                                                                      spec.roi_levels[0], spec.roi_levels[-1]),
                                             cfg.KRCNN.NUM_STACKED_CONVS)
                h = npy(h)
                maps.append(flip_heatmaps(h, plan.perm) if v.flip else h)
            heat = combine(np.stack(maps), plan.hm_max)
            keyps = okp.keypoint_results(heat, det_boxes, K)
    return dict(cls_boxes=cls_boxes[1], cls_boxes_all=cls_boxes, keyps=keyps, heat=heat, union_count=union_count)
