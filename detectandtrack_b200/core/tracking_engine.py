"""Per-video detection linking on the GPU — drop-in for the default path of the
reference's ``core.tracking_engine`` (lib/core/tracking_engine.py).

Kept surface: ``_compute_matches``, ``_compute_tracks_video``,
``compute_matches_tracks``, ``_prune_bad_detections``, ``_center_detections``,
``run_posetrack_tracking`` with the reference's argument meaning and the
``detections.pkl`` / ``detections_withTracks.pkl`` schema; the PoseTrack JSON
writer that follows it lives in ``core/mpii_eval_engine.py``.

What changed underneath: instead of one python loop per frame pair
(bbox_overlaps -> scipy LSA -> id list), all frames of all videos are packed
into one [F, Dmax, 4T+1] tensor and three launches do the work
(csrc/lsa.cu): fused (1 - IoU) cost + assignment for every consecutive pair
(pairs are independent), then the sequential id scan, one thread per video.
Only the 'bbox-overlap' cost runs on the device (the configuration of every shipped yaml; the
weights of the other costs are 0, config.py:550-551), with 'hungarian' or 'greedy' matching;
anything else raises NotImplementedError.

TRACKING.DEBUG.UPPER_BOUND / _2_GT_KPS / _5_GT_KPS_ONLY (:282-338), the upper-bound experiments, match the GT of every frame
against its detections in one batched pass over the frames interleaved with their GT (csrc/upper_bound.cu), then one
launch keeps the matched detections with the GT's track ids and copies the GT's boxes and keypoints onto them.

TRACKING.FLOW_SMOOTHING_ON (:401-643) runs after the id pass, one video at a time: Farneback flow
between consecutive key frames (csrc/flow.cu, all pairs of a frame size in one call), the shot-boundary
test np.abs(flow).mean() > FLOW_SHOT_BOUNDARY_TH on the device, then one launch that shifts every pose
±N_CONTEXT_FRAMES along the flow and combines the shifts per track.  Only the output track order of each
frame (the reference's list(set(...)), CPython's set order) is computed on the host.
"""
import logging
import os.path as osp
import pickle

import numpy as np

from .config import cfg
from ..ops import box_ops

logger = logging.getLogger(__name__)

MAX_TRACK_IDS = box_ops.MAX_TRACK_IDS      # tracking_engine.py:45
FIRST_TRACK_ID = box_ops.FIRST_TRACK_ID    # tracking_engine.py:46


# ----------------------------------------------------------------- file I/O
def _load_det_file(det_fpath):
    with open(det_fpath, 'rb') as fin:
        try:
            return pickle.load(fin)
        except UnicodeDecodeError:          # pickles written by the py2 reference
            fin.seek(0)
            return pickle.load(fin, encoding='latin1')


def _write_det_file(dets, det_fpath):
    with open(det_fpath, 'wb') as fout:
        pickle.dump(dets, fout, pickle.HIGHEST_PROTOCOL)


def _image_path(entry):
    """lib/utils/image.py:44-48 get_image_path: the CENTRE frame of a clip entry."""
    im = entry['image']
    return im[len(im) // 2] if isinstance(im, (list, tuple)) else im


def _is_same_video(json1, json2):
    return osp.dirname(_image_path(json1)) == osp.dirname(_image_path(json2))


def _get_boxes(dets, img_id):
    return dets['all_boxes'][1][img_id]


def _get_poses(dets, img_id):
    return dets['all_keyps'][1][img_id]


# ------------------------------------------------------- centre / prune (host)
def _center_boxes(boxes):
    """:86-93"""
    if len(boxes) == 0:
        return boxes
    assert (boxes.shape[-1] - 1) % 4 == 0, 'Must contain scores in last col.'
    time_dim = (boxes.shape[-1] - 1) // 4
    center = time_dim // 2
    return boxes[:, np.array(list(range(center * 4, (center + 1) * 4)) + [-1])]


def _center_poses(poses):
    """:96-103"""
    if len(poses) == 0:
        return poses
    K = cfg.KRCNN.NUM_KEYPOINTS
    time_dim = poses[0].shape[-1] // K
    center = time_dim // 2
    return [el[..., center * K:(center + 1) * K] for el in poses]


def _center_detections(dets):
    """:751-755"""
    for img_id in range(len(dets['all_boxes'][1])):
        dets['all_boxes'][1][img_id] = _center_boxes(_get_boxes(dets, img_id))
        dets['all_keyps'][1][img_id] = _center_poses(_get_poses(dets, img_id))


def _pack(box_list, ld=None):
    """list of (n_i, ld) arrays -> padded [F, Dmax, ld] fp32 + counts."""
    F = len(box_list)
    counts = np.array([0 if b is None else len(b) for b in box_list], dtype=np.int32)
    if ld is None:
        ld = max([b.shape[1] for b in box_list if b is not None and len(b)] + [5])
    dmax = max(int(counts.max()) if F else 0, 1)
    packed = np.zeros((F, dmax, ld), dtype=np.float32)
    for i, b in enumerate(box_list):
        if counts[i]:
            packed[i, :counts[i]] = b
    return packed, counts


def _prune_bad_detections(dets, json_data, conf):
    """:731-748 on the device for all images at once (dt_prune_detections).
    Like the reference, the kept boxes are the clipped ones."""
    import torch
    boxes_l = dets['all_boxes'][1]
    N = len(boxes_l)
    if N == 0:
        return dets
    packed, counts = _pack(boxes_l)
    T = (packed.shape[2] - 1) // 4
    hw = np.array([[json_data[i]['height'], json_data[i]['width']] for i in range(N)], dtype=np.float32)
    out, counts_out, sel = box_ops.prune_detections(
        torch.from_numpy(packed).cuda(), torch.from_numpy(counts), torch.from_numpy(hw),
        conf, T=T, center_only=False)
    out, counts_out, sel = out.cpu().numpy(), counts_out.cpu().numpy(), sel.cpu().numpy()
    for i in range(N):
        n = int(counts_out[i])
        poses = dets['all_keyps'][1][i]
        dets['all_boxes'][1][i] = out[i, :n].copy()
        dets['all_keyps'][1][i] = [poses[j] for j in sel[i, :n].tolist()]
    return dets


# ------------------------------------------------------------------ matching
POSETRACK_KEYPOINTS = ['nose', 'head_bottom', 'head_top', 'left_ear', 'right_ear', 'left_shoulder', 'right_shoulder', 'left_elbow',
                       'right_elbow', 'left_wrist', 'right_wrist', 'left_hip', 'right_hip', 'left_knee', 'right_knee', 'left_ankle',
                       'right_ankle']          # person_cat_info['keypoints'] of the PoseTrack json datasets


def _cost_weights(cost_types, cost_weights):
    """(w_iou, w_pck) of TRACKING.DISTANCE_METRICS / _WTS (tracking_engine.py:158-181); 'cnn-cosdist' needs a CNN feature
    extractor (utils/pytorch_cnn_features, weight 0 in every shipped yaml) and is not on the device path."""
    assert len(cost_weights) == len(cost_types)
    w = {'bbox-overlap': 0.0, 'pose-pck': 0.0}
    for t, wt in zip(cost_types, cost_weights):
        if wt == 0:
            continue
        if t not in w:
            raise NotImplementedError('device tracking implements the bbox-overlap and pose-pck costs (got %r)' % (t,))
        w[t] += float(wt)
    if w['bbox-overlap'] == 0.0 and w['pose-pck'] == 0.0:
        raise NotImplementedError('no active tracking cost')
    return w['bbox-overlap'], w['pose-pck']


def _check_default_cost(cost_types, cost_weights):
    w_iou, w_pck = _cost_weights(cost_types, cost_weights)
    if w_pck != 0.0:
        raise NotImplementedError('this call path takes boxes only; pose-pck needs the poses (see _tracks_for_videos)')
    return w_iou


def _pack_poses(pose_list, dmax, K):
    """list (frames) of lists of [4|3, K] arrays -> [F, dmax, 4, K] fp32 (x row, y row used by the cost)."""
    out = np.zeros((len(pose_list), dmax, 4, K), dtype=np.float32)
    for f, poses in enumerate(pose_list):
        for i, p in enumerate(poses or []):
            p = np.asarray(p, dtype=np.float32)
            out[f, i, :p.shape[0]] = p
    return out


def _compute_matches(prev_frame_data, cur_frame_data, prev_boxes, cur_boxes,
                     prev_poses, cur_poses, cost_types, cost_weights,
                     bipart_match_algo, C=None):
    """:209-246.  Returns int32 matches[n_cur] = index into prev boxes, or -1."""
    import torch
    if bipart_match_algo not in box_ops.ALGOS:
        raise NotImplementedError('Unknown matching algo: {}'.format(bipart_match_algo))
    if C is not None:
        # scipy solves the matrix in fp64: a float32 one is exact in fp32, any other is solved in fp64
        C = np.ascontiguousarray(C, dtype=np.float32 if np.asarray(C).dtype == np.float32 else np.float64)
        P, Q = C.shape
        if P == 0 or Q == 0:
            return -np.ones((Q,), dtype=np.int32)
        m, status = box_ops.lsa_batched(torch.from_numpy(C).cuda().unsqueeze(0),
                                        torch.tensor([P]), torch.tensor([Q]), bipart_match_algo)
        _check_status(status)
        return m[0, :Q].cpu().numpy().astype(np.int32)
    weight = _check_default_cost(cost_types, cost_weights)
    nboxes = cur_boxes.shape[0]
    if nboxes == 0 or prev_boxes.shape[0] == 0:
        return -np.ones((nboxes,), dtype=np.int32)
    packed, counts = _pack([prev_boxes, cur_boxes])
    T = (packed.shape[2] - 1) // 4
    m, _ = box_ops.match_frames(torch.from_numpy(packed).cuda(), torch.from_numpy(counts), None, T=T, weight=weight,
                                algo=bipart_match_algo)
    return m[1, :nboxes].cpu().numpy().astype(np.int32)


def _check_status(*statuses):
    """scipy's ValueError for a cost matrix it cannot solve: the solver's status 1 (infeasible, or a NaN / -inf entry)."""
    for st in statuses:
        if st is not None and bool(st.cpu().numpy().any()):
            raise ValueError('cost matrix is infeasible or contains invalid numeric entries')


def _pose_cost_args(videos_poses, kpt_names=None):
    names = list(kpt_names or POSETRACK_KEYPOINTS)
    K = cfg.KRCNN.NUM_KEYPOINTS
    if K <= 0:                                   # unset (config default -1): take it from the data
        K = next((np.asarray(p).shape[-1] for vp in videos_poses for fr in vp for p in (fr or [])), len(names))
    return K, names.index('head_top'), names.index('head_bottom')


def _tracks_for_videos(videos_boxes, videos_poses=None, kpt_names=None, videos_prev_poses=None):
    """videos_boxes: list (videos) of lists (frames) of (n,4T+1) arrays; videos_poses (needed when the 'pose-pck' cost is
    active): same nesting of lists of [4, K] keypoint arrays.  videos_prev_poses (same nesting, or None): the poses frame f
    shows as the previous frame of f + 1 when they differ from its own (UPPER_BOUND_5_GT_KPS_ONLY replaces them after the
    match, :325-338).  Returns list of list of python-int id lists, one batched device pass."""
    import torch
    flat, first = [], []
    for vb in videos_boxes:
        first.append(len(flat))
        flat.extend(vb)
    if not flat:
        return [[] for _ in videos_boxes]
    packed, counts = _pack(flat)
    T = (packed.shape[2] - 1) // 4
    is_start = np.zeros(len(flat), dtype=np.uint8)
    is_start[np.array(first, dtype=np.int64)] = 1
    w_iou, w_pck = _cost_weights(cfg.TRACKING.DISTANCE_METRICS, cfg.TRACKING.DISTANCE_METRIC_WTS)
    algo = cfg.TRACKING.BIPARTITE_MATCHING_ALGO
    if algo not in box_ops.ALGOS:
        raise NotImplementedError('Unknown matching algo: {}'.format(algo))
    d_counts = torch.from_numpy(counts).cuda()
    d_start = torch.from_numpy(is_start).cuda()
    if w_pck == 0.0:
        matches, status = box_ops.match_frames(torch.from_numpy(packed).cuda(), d_counts, d_start, T=T, weight=w_iou, algo=algo)
    elif videos_prev_poses is not None:
        matches, status = _pair_matches(flat, first, videos_poses, videos_prev_poses, packed.shape[1], w_iou, w_pck, algo, kpt_names)
    else:
        # combined cost (tracking_engine.py:158-181): cost matrices of every frame pair in one launch, then the batched solver
        assert videos_poses is not None, "the 'pose-pck' cost needs the poses of every detection"
        K, ht, hb = _pose_cost_args(videos_poses, kpt_names)
        poses = _pack_poses([p for vp in videos_poses for p in vp], packed.shape[1], K)
        cost = box_ops.frame_costs(torch.from_numpy(packed).cuda(), d_counts, d_start, torch.from_numpy(poses).cuda(), T=T, w_iou=w_iou,
                                   w_pck=w_pck, head_top=ht, head_bottom=hb)
        nrows = torch.cat([d_counts[:1] * 0, d_counts[:-1]]) * (1 - d_start.to(torch.int32))
        matches, status = box_ops.lsa_batched(cost, nrows, d_counts, algo)
    tracks = box_ops.assign_track_ids(matches, d_counts, torch.tensor(first, dtype=torch.int32), d_start)
    tracks = tracks.cpu().numpy()
    _check_status(status)
    out = []
    for v, vb in enumerate(videos_boxes):
        f0 = first[v]
        out.append([tracks[f0 + i, :counts[f0 + i]].tolist() for i in range(len(vb))])
    return out


def _pair_matches(flat, first, videos_poses, videos_prev_poses, dmax, w_iou, w_pck, algo, kpt_names=None):
    """The combined cost of every frame pair (f - 1, f) of every video with frame f - 1's poses taken from
    videos_prev_poses: the pairs are packed pair-interleaved, [(f - 1, f), ...] with is_start on every first entry, for
    dt_frame_costs + dt_lsa_batched_f64.  Returns matches [F, dmax] in frame order (first frames of videos: -1) and the
    solver's status per pair (None without pairs)."""
    import torch
    F = len(flat)
    cur = [p for vp in videos_poses for p in vp]
    prev = [p for vp in videos_prev_poses for p in vp]
    is_first = np.zeros(F, dtype=bool)
    is_first[np.array(first, dtype=np.int64)] = True
    pair_of = [f for f in range(F) if not is_first[f]]
    out = torch.full((F, dmax), -1, dtype=torch.int32, device='cuda')
    if not pair_of:
        return out, None
    boxes, pposes = [], []
    for f in pair_of:
        boxes += [flat[f - 1], flat[f]]
        pposes += [prev[f - 1], cur[f]]
    packed, counts = _pack(boxes)
    T = (packed.shape[2] - 1) // 4
    K, ht, hb = _pose_cost_args([pposes], kpt_names)
    poses = _pack_poses(pposes, packed.shape[1], K)
    is_start = np.zeros(len(boxes), dtype=np.uint8)
    is_start[0::2] = 1
    d_counts = torch.from_numpy(counts).cuda()
    cost = box_ops.frame_costs(torch.from_numpy(packed).cuda(), d_counts, torch.from_numpy(is_start).cuda(),
                               torch.from_numpy(poses).cuda(), T=T, w_iou=w_iou, w_pck=w_pck, head_top=ht, head_bottom=hb)
    nrows = torch.cat([d_counts[:1] * 0, d_counts[:-1]]) * (1 - torch.from_numpy(is_start).cuda().to(torch.int32))
    m, status = box_ops.lsa_batched(cost, nrows, d_counts, algo)
    w = min(dmax, m.shape[1])
    out[torch.tensor(pair_of, device='cuda'), :w] = m[1::2, :w]
    return out, status


# ------------------------------------------------------------------------------ upper-bound experiments
def _gt_arrays(entry, i, T):
    """The GT of a roidb entry as the reference's roidb holds it: boxes [G, 4T] fp32, gt_keypoints [G, 3, K] int32 (json_dataset
    stores the annotation's coordinates in an int32 array, truncating them; a JSON-list roidb hands them over as they are in
    the file), tracks [G]."""
    for k in ('boxes', 'gt_keypoints', 'tracks'):
        if k not in entry:
            raise ValueError("TRACKING.DEBUG.UPPER_BOUND*: roidb entry %d (%s) has no ground truth '%s'" % (i, _image_path(entry), k))
    boxes = np.asarray(entry['boxes'], dtype=np.float32)
    boxes = boxes.reshape(-1, boxes.shape[-1]) if boxes.size else np.zeros((0, 4 * T), np.float32)
    kps = np.asarray(entry['gt_keypoints']).astype(np.int32)
    tracks = np.asarray(entry['tracks']).reshape(-1)
    if len(tracks) != len(boxes) or (kps.size and kps.shape[0] != len(boxes)):
        raise ValueError('roidb entry %d: %d GT boxes, %d keypoint sets and %d track ids' % (i, len(boxes), len(kps), len(tracks)))
    if boxes.shape[1] != 4 * T:
        raise NotImplementedError('TRACKING.DEBUG.UPPER_BOUND*: roidb entry %d has GT boxes of %d columns for detections of '
                                  '%d frame(s)' % (i, boxes.shape[1], T))
    return boxes, kps, tracks


def _box_frames(dets):
    """T of the detections (4T + 1 box columns)."""
    ld = next((np.shape(b)[-1] for b in dets['all_boxes'][1] if len(b)), 5)
    return (ld - 1) // 4


def _check_upper_bound_options(json_data=None, dets=None):
    """Rejects, before any device work, the upper-bound modes the device path does not run and a roidb without the GT
    they read."""
    dbg = cfg.TRACKING.DEBUG
    if dbg.UPPER_BOUND_3_SHOTS:
        raise NotImplementedError('TRACKING.DEBUG.UPPER_BOUND_3_SHOTS reads a hard-coded shot-boundary file '
                                  '(/path/to/shot_boundaries_val.csv, :258-271) that is not part of the release')
    if not (dbg.UPPER_BOUND or dbg.UPPER_BOUND_5_GT_KPS_ONLY) or json_data is None:
        return
    T = _box_frames(dets)
    if dbg.UPPER_BOUND and dbg.UPPER_BOUND_2_GT_KPS and T > 1:
        raise NotImplementedError('TRACKING.DEBUG.UPPER_BOUND_2_GT_KPS sets new_boxes[:, :4] from the GT (:313), which '
                                  'takes centre-frame boxes (T = 1); the detections have T = %d' % T)
    for i, entry in enumerate(json_data):
        _gt_arrays(entry, i, T)


def _upper_bound_tracks(all_video_roidb, dets):
    """:282-338 for every video in one batched device pass.  Replaces the boxes / poses of dets as the reference does and
    returns the per-video lists of per-frame id lists (the GT track ids under UPPER_BOUND, else the regular id pass over
    the frames, with the _5 poses of frame f - 1 in the pose-pck cost of the pair (f - 1, f))."""
    import torch
    dbg = cfg.TRACKING.DEBUG
    ub, ub2, conf_only, ub5 = dbg.UPPER_BOUND, dbg.UPPER_BOUND_2_GT_KPS, dbg.UPPER_BOUND_2_GT_KPS_ONLY_CONF, dbg.UPPER_BOUND_5_GT_KPS_ONLY
    frames = [e for v in all_video_roidb for e in v]
    F = len(frames)
    if F == 0:
        return [[] for _ in all_video_roidb]
    boxes = [_get_boxes(dets, det_id) for (_, det_id) in frames]
    poses = [_get_poses(dets, det_id) for (_, det_id) in frames]
    T = _box_frames(dets)
    ld = 4 * T + 1
    w_iou, w_pck = _cost_weights(cfg.TRACKING.DISTANCE_METRICS, cfg.TRACKING.DISTANCE_METRIC_WTS)
    algo = cfg.TRACKING.BIPARTITE_MATCHING_ALGO
    if algo not in box_ops.ALGOS:
        raise NotImplementedError('Unknown matching algo: {}'.format(algo))
    gts = [_gt_arrays(e, det_id, T) for (e, det_id) in frames]
    stacked = [np.stack(ps).astype(np.float32, copy=False) if len(ps) else None for ps in poses]
    shapes = {p.shape[1:] for p in stacked if p is not None}
    if len(shapes) > 1:
        raise NotImplementedError('detection poses of different shapes: %s' % sorted(shapes))
    R, K = shapes.pop() if shapes else (4, max([g[1].shape[-1] for g in gts if g[1].size] + [17]))
    if R < 3:
        raise NotImplementedError('detection poses of %d rows: the GT replaces rows 0..2' % R)
    for i, (_, kp, _) in enumerate(gts):
        if kp.size and kp.shape[1:] != (3, K):
            raise NotImplementedError('roidb entry %d: GT keypoints %s for detection poses [%d, %d]'
                                      % (frames[i][1], kp.shape, R, K))
    dmax = max([len(b) for b in boxes] + [len(g[0]) for g in gts] + [1])
    if dmax > box_ops.L.LSA_MAX_DIM:
        raise ValueError('TRACKING.DEBUG.UPPER_BOUND*: %d GT people or detections in a frame (at most %d)'
                         % (dmax, box_ops.L.LSA_MAX_DIM))
    pb = np.zeros((2 * F, dmax, ld), np.float32)
    pp = np.zeros((2 * F, dmax, R, K), np.float32)
    cnt = np.zeros(2 * F, np.int32)
    tid = np.full((F, dmax), -1, np.int32)
    for f in range(F):
        gb, gk, gt = gts[f]
        cnt[2 * f], cnt[2 * f + 1] = len(gb), len(boxes[f])
        pb[2 * f, :len(gb), :4 * T] = gb
        if gk.size:
            pp[2 * f, :len(gk), :3] = gk
        tid[f, :len(gt)] = gt
        if len(boxes[f]):
            pb[2 * f + 1, :len(boxes[f])] = boxes[f]
        if stacked[f] is not None:
            pp[2 * f + 1, :len(stacked[f])] = stacked[f]
    is_start = np.zeros(2 * F, np.uint8)
    is_start[0::2] = 1
    d_b, d_p, d_n = torch.from_numpy(pb).cuda(), torch.from_numpy(pp).cuda(), torch.from_numpy(cnt).cuda()
    d_s = torch.from_numpy(is_start).cuda()
    matches = matches_gt = status = status_gt = None
    if ub:
        if w_pck == 0.0:
            matches, status = box_ops.match_frames(d_b, d_n, d_s, T=T, weight=w_iou, algo=algo)
        else:
            _, ht, hb = _pose_cost_args([poses])
            cost = box_ops.gt_frame_costs(d_b, d_n, d_p, T=T, w_iou=w_iou, w_pck=w_pck, head_top=ht, head_bottom=hb)
            matches, status = box_ops.lsa_batched(cost, d_n[0::2], d_n[1::2], algo)
    if ub5:                                                   # bbox-overlap, weight 1, hungarian (:329-333)
        matches_gt, status_gt = box_ops.match_frames(d_b, d_n, d_s, T=T, weight=1.0, algo='hungarian')
    _check_status(status, status_gt)
    flags = (box_ops.L.UB_COMPACT if ub else 0) | (box_ops.L.UB_GT_KPS if ub and ub2 else 0) | \
        (box_ops.L.UB_ONLY_CONF if ub and ub2 and conf_only else 0)
    ob, op, ot, on = box_ops.track_upper_bound(d_b, d_p, d_n, torch.from_numpy(tid).cuda(), matches, matches_gt, flags)
    ob, op, ot, on = ob.cpu().numpy(), op.cpu().numpy(), ot.cpu().numpy(), on.cpu().numpy()
    new_poses = []
    for f, (_, det_id) in enumerate(frames):
        n = int(on[f])
        dets['all_boxes'][1][det_id] = ob[f, :n].copy()
        new_poses.append(list(op[f, :n].copy()))
        dets['all_keyps'][1][det_id] = new_poses[-1]
    out, f0 = [], 0
    if ub:
        for v in all_video_roidb:
            out.append([ot[f, :int(on[f])].tolist() for f in range(f0, f0 + len(v))])
            f0 += len(v)
        return out
    vb, vp, vq = [], [], []
    for v in all_video_roidb:
        vb.append(boxes[f0:f0 + len(v)]); vp.append(poses[f0:f0 + len(v)]); vq.append(new_poses[f0:f0 + len(v)])
        f0 += len(v)
    return _tracks_for_videos(vb, vp, videos_prev_poses=vq)


def _compute_tracks_video(video_json_data, dets):
    """:272-350 for one video: list of per-frame id lists (the TRACKING.DEBUG.UPPER_BOUND* modes replace the video's
    boxes and poses in dets, as the reference does)."""
    _check_upper_bound_options([e for e, _ in video_json_data], dets)
    if cfg.TRACKING.DEBUG.UPPER_BOUND or cfg.TRACKING.DEBUG.UPPER_BOUND_5_GT_KPS_ONLY:
        return _upper_bound_tracks([video_json_data], dets)[0]
    boxes = [_get_boxes(dets, det_id) for (_, det_id) in video_json_data]
    poses = [_get_poses(dets, det_id) for (_, det_id) in video_json_data]
    return _tracks_for_videos([boxes], [poses])[0]


# ------------------------------------------------------------------------------ flow smoothing
def _check_tracking_options(dets, json_data=None):
    """Rejects, before any device work, what the device path does not run: LSTM tracking, and flow smoothing with
    anything but centre-frame boxes (T = 1) and [4, 17] poses (the shapes _weighted_avg_poses and _combine_boxes
    take, :454-479) or with the FLOW_SMOOTHING_COMBINE debugger hook."""
    if cfg.TRACKING.LSTM_TEST.LSTM_TRACKING_ON:
        raise NotImplementedError('LSTM tracking is outside the device path')
    _check_upper_bound_options(json_data, dets)
    if not cfg.TRACKING.FLOW_SMOOTHING_ON:
        return
    if cfg.TRACKING.DEBUG.FLOW_SMOOTHING_COMBINE:
        raise NotImplementedError('TRACKING.DEBUG.FLOW_SMOOTHING_COMBINE (a pdb hook) is not on the device path')
    n = cfg.TRACKING.FLOW_SMOOTHING.N_CONTEXT_FRAMES
    assert n >= 0                                                   # :612
    if n > FLOW_MAX_CONTEXT:
        raise NotImplementedError('N_CONTEXT_FRAMES=%d exceeds %d' % (n, FLOW_MAX_CONTEXT))
    for i, b in enumerate(dets['all_boxes'][1]):
        if len(b) and np.shape(b)[-1] != 5:
            raise NotImplementedError('flow smoothing takes centre-frame boxes (4T+1 = 5 columns); image %d has %d'
                                      % (i, np.shape(b)[-1]))
    for i, ps in enumerate(dets['all_keyps'][1]):
        for p in ps:
            if np.shape(p) != (4, 17):
                raise NotImplementedError('flow smoothing takes [4, 17] poses (17 centre-frame joints); image %d has %s'
                                          % (i, np.shape(p)))


FLOW_MAX_CONTEXT = 16        # DT_FLOW_MAX_CONTEXT of include/dt_b200.h
FLOW_MAX_PAIRS = 32          # pairs per dt_farneback_flow call (bounds the memory: about 90 MB per 720p pair)


def read_key_frame(entry):
    """lib/utils/image.py:65-79 read_image_video(entry, key_frame_only=True): the centre frame of a clip entry
    (get_image_path, :44-48) as BGR uint8.  Synthetic entries take test_engine's seeded frame of that index."""
    if entry.get('synthetic'):
        from .test_engine import _synthetic_frame
        T = cfg.VIDEO.NUM_FRAMES if cfg.MODEL.VIDEO_ON else 1
        return _synthetic_frame(entry['height'], entry['width'], entry['seed'], T // 2)
    import cv2
    path = _image_path(entry)
    im = cv2.imread(path)
    assert im is not None, 'could not read {}'.format(path)
    return im


def _read_key_frames(video_json_data):
    """read_key_frame of every entry, on loader threads."""
    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(max_workers=8) as ex:
        return list(ex.map(lambda e: np.ascontiguousarray(read_key_frame(e[0]), dtype=np.uint8), video_json_data))


def compute_optical_flow(video_json_data):
    """:573-597.  Returns (flows, means): flows[i] the cuda fp32 [H, W, 2] flow of key frame i -> i + 1 (None for a
    pair of different frame sizes, where cv2 raises), means[i] = np.abs(flows[i]).mean() as np.float32."""
    import torch
    from ..ops import flow_ops
    frames = _read_key_frames(video_json_data)
    n = len(frames)
    flows, means = [None] * max(n - 1, 0), [None] * max(n - 1, 0)
    i = 0
    while i < n - 1:
        j = i                                  # frames i..j share one size; pairs i..j-1 go to the device in chunks
        while j + 1 < n and frames[j + 1].shape == frames[i].shape:
            j += 1
        for a in range(i, j, FLOW_MAX_PAIRS):
            b = min(a + FLOW_MAX_PAIRS, j)
            clip = torch.from_numpy(np.stack(frames[a:b + 1])).cuda()
            f = flow_ops.farneback_flow(clip, [(k, k + 1) for k in range(b - a)])
            m = flow_ops.flow_mean_abs(f).cpu().numpy()
            for k in range(b - a):
                flows[a + k], means[a + k] = f[k], m[k]
        i = j + 1
    return flows, means


def _output_tracks(tracks, counts, moves, n_context, extend):
    """The track list of every frame after _combine_shifted_poses (:491-498): shift s of frame f holds the tracks of
    frame f - s when that frame has detections and the chain of pairs between them moves (``moves[q]``: the pair
    q -> q + 1 has a flow below the shot-boundary threshold)."""
    n = len(tracks)
    out = []
    for f in range(n):
        if not extend:
            out.append(list(tracks[f]))
            continue
        ids = set()
        for s in range(-n_context, n_context + 1):
            g = f - s
            if 0 <= g < n and counts[g] and all(moves[q] for q in range(min(g, f), max(g, f))):
                ids |= set(tracks[g])
        out.append(list(ids))
    return out


def _smooth_pose_video(video_json_data, dets, tracks):
    """:600-643.  Replaces the poses and boxes of the video's images with the flow-smoothed ones and returns the
    new per-frame track lists."""
    import torch
    from ..ops import flow_ops
    ncontext = cfg.TRACKING.FLOW_SMOOTHING.N_CONTEXT_FRAMES
    assert ncontext >= 0
    n = len(video_json_data)
    if n == 0:
        return []
    poses = [_get_poses(dets, det_id) for (_, det_id) in video_json_data]
    boxes = [_get_boxes(dets, det_id) for (_, det_id) in video_json_data]
    counts = [len(t) for t in tracks]
    for f in range(n):
        assert len(poses[f]) == len(boxes[f]) == counts[f], 'frame %d: poses, boxes and tracks differ in number' % f
    flows, moves = [None] * n, [False] * n
    if ncontext > 0 and n > 1:
        fl, means = compute_optical_flow(video_json_data)
        th = cfg.TRACKING.FLOW_SMOOTHING.FLOW_SHOT_BOUNDARY_TH
        for q in range(n - 1):
            flows[q] = fl[q]
            moves[q] = fl[q] is not None and not (means[q] > th)        # :404-407
    out_tracks = _output_tracks(tracks, counts, moves, ncontext, cfg.TRACKING.FLOW_SMOOTHING.EXTEND_TRACKS)
    dmax = max(max(counts), 1)
    packed_b, _ = _pack(boxes, ld=5)
    packed_p = _pack_poses(poses, dmax, 17)
    packed_t = np.full((n, dmax), -1, dtype=np.int32)
    for f in range(n):
        packed_t[f, :counts[f]] = tracks[f]
    ocounts = np.array([len(t) for t in out_tracks], dtype=np.int32)
    omax = max(int(ocounts.max()), 1)
    packed_o = np.zeros((n, omax), dtype=np.int32)
    for f in range(n):
        packed_o[f, :ocounts[f]] = out_tracks[f]
    is_start = np.zeros(n, dtype=np.uint8)
    is_start[0] = 1
    p, b = flow_ops.smooth_poses(packed_p, packed_b[:, :dmax], counts, packed_t, is_start, flows,
                                 np.array([not m for m in moves], dtype=np.uint8), ncontext, packed_o, ocounts)
    p, b = p.cpu().numpy(), b.cpu().numpy()
    for f, (_, det_id) in enumerate(video_json_data):
        k = int(ocounts[f])
        dets['all_keyps'][1][det_id] = [p[f, o].copy() for o in range(k)]
        # a frame left without tracks gets np.zeros((0, box_size)), fp64 as in the reference (:541-544)
        dets['all_boxes'][1][det_id] = b[f, :k].copy() if k else np.zeros((0, boxes[f].shape[-1]))
    return out_tracks


def compute_matches_tracks(json_data, dets, lstm_model=None):
    """:669-708.  Splits images into videos by dirname, links every video in one
    batched device pass, writes dets['all_tracks'] = [[], per-image id lists].
    With TRACKING.FLOW_SMOOTHING_ON each video's poses and boxes are then smoothed along the flow (:695-697)."""
    _check_tracking_options(dets, json_data)
    num_imgs = len(json_data)
    all_tracks = [[]] * num_imgs
    all_video_roidb, video_entries = [], []
    for img_id in range(num_imgs):
        if img_id == 0 or _is_same_video(json_data[img_id - 1], json_data[img_id]):
            video_entries.append((json_data[img_id], img_id))
        else:
            all_video_roidb.append(sorted(video_entries, key=lambda x: _image_path(x[0])))
            video_entries = [(json_data[img_id], img_id)]
    if len(video_entries) > 0:
        all_video_roidb.append(video_entries)
    assert num_imgs == sum(len(v) for v in all_video_roidb)
    logger.info('Computing tracks for %d videos.', len(all_video_roidb))
    if cfg.TRACKING.DEBUG.UPPER_BOUND or cfg.TRACKING.DEBUG.UPPER_BOUND_5_GT_KPS_ONLY:
        tracks = _upper_bound_tracks(all_video_roidb, dets)
    else:
        vids = [[_get_boxes(dets, det_id) for (_, det_id) in v] for v in all_video_roidb]
        vposes = [[_get_poses(dets, det_id) for (_, det_id) in v] for v in all_video_roidb]
        tracks = _tracks_for_videos(vids, vposes)
    if cfg.TRACKING.FLOW_SMOOTHING_ON:
        tracks = [_smooth_pose_video(entries, dets, tracks[v]) for v, entries in enumerate(all_video_roidb)]
    for v, entries in enumerate(all_video_roidb):
        for i, (_, det_id) in enumerate(entries):
            all_tracks[det_id] = tracks[v][i]
    dets['all_tracks'] = [[], all_tracks]
    return dets


def run_posetrack_tracking(test_output_dir, json_data, write_json=True, dataset=None):
    """:758-795.  Writes detections_withTracks.pkl and then, like the reference's run_mpii_eval call
    (:792-795), the per-video PoseTrack JSON files (core/mpii_eval_engine.py).  With a dataset whose
    annotation_directory is set (EVAL.POSETRACK_ANNOTATION_DIR), they are then scored against it."""
    det_file = cfg.TRACKING.DETECTIONS_FILE if len(cfg.TRACKING.DETECTIONS_FILE) else \
        osp.join(test_output_dir, 'detections.pkl')
    out_det_file = osp.join(test_output_dir, 'detections_withTracks.pkl')
    if not osp.exists(det_file):
        raise ValueError('Output file not found {}'.format(det_file))
    logger.info('Tracking over %s', det_file)
    if cfg.TRACKING.DEBUG.UPPER_BOUND_2_GT_KPS:        # :770-771
        cfg.TRACKING.DEBUG.UPPER_BOUND = True
    dets = _load_det_file(det_file)
    if cfg.TRACKING.KEEP_CENTER_DETS_ONLY:
        _center_detections(dets)
    assert len(json_data) == len(dets['all_boxes'][1])
    assert len(json_data) == len(dets['all_keyps'][1])
    _check_tracking_options(dets, json_data)
    conf = cfg.TRACKING.CONF_FILTER_INITIAL_DETS
    logger.info('Pruning detections with less than %s confidence', conf)
    dets = _prune_bad_detections(dets, json_data, conf)
    dets_withTracks = compute_matches_tracks(json_data, dets, None)
    _write_det_file(dets_withTracks, out_det_file)
    if write_json:
        from . import mpii_eval_engine
        mpii_eval_engine.run_mpii_eval(test_output_dir, json_data, dataset)
    return dets_withTracks
