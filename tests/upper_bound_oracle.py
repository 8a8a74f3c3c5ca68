"""CPU restatement of the upper-bound experiments (TEST INFRASTRUCTURE ONLY), on top of the oracle package:

  tracking_engine._compute_tracks_video (:272-350) with TRACKING.DEBUG.UPPER_BOUND / _2_GT_KPS / _2_GT_KPS_ONLY_CONF /
  _5_GT_KPS_ONLY, costs of _compute_distance_matrix (:158-181) with oracle.boxes / oracle.keypoints, scipy's
  linear_sum_assignment or oracle.lsa's greedy matcher   -> compute_tracks_video
  poseval's assignGTmulti(..., computeUpperBound=True) (eval_helpers.py:423-637, the MOT inputs only), then
  oracle.poseval's MOTAccumulator and computeMetrics     -> evaluate_tracking_upper_bound

The reference's in-place pose writes are kept as aliasing of numpy arrays, as the reference has them."""
import math

import numpy as np
import scipy.optimize

from oracle import boxes as obox
from oracle import keypoints as okps
from oracle import poseval as ope
from oracle.lsa import bipartite_matching_greedy

POSETRACK_KEYPOINTS = ['nose', 'head_bottom', 'head_top', 'left_ear', 'right_ear', 'left_shoulder', 'right_shoulder',
                       'left_elbow', 'right_elbow', 'left_wrist', 'right_wrist', 'left_hip', 'right_hip', 'left_knee',
                       'right_knee', 'left_ankle', 'right_ankle']
MAX_TRACK_IDS = 999


def compute_matches(prev_boxes, cur_boxes, prev_poses, cur_poses, w_iou, w_pck, algo):
    """:158-246 -> matches[q] = previous row or -1 (int32)."""
    Cs = []
    if w_iou != 0:
        C = 1 - obox.bbox_overlaps(prev_boxes, cur_boxes)            # fp32, scaled in place as the reference does
        C *= w_iou
        Cs.append(C)
    if w_pck != 0:
        C = okps.pairwise_kpt_distance(prev_poses, cur_poses, POSETRACK_KEYPOINTS)
        C *= w_pck
        Cs.append(C)
    C = np.sum(np.stack(Cs, axis=0), axis=0)
    matches = -np.ones((cur_boxes.shape[0],), dtype=np.int32)
    if algo == 'hungarian':
        p, q = scipy.optimize.linear_sum_assignment(C)
    else:
        p, q = bipartite_matching_greedy(C)
    for a, b in zip(p, q):
        matches[b] = a
    return matches


def compute_tracks_video(frames, ub, ub2, conf_only, ub5, w_iou=1.0, w_pck=0.0, algo='hungarian'):
    """frames: list of dicts boxes [n, 5] fp32, poses (list of [4, K] fp32), gt_boxes [G, 4] fp32, gt_kps [G, 3, K] int32,
    gt_tracks [G].  Returns (boxes per frame, poses per frame, track ids per frame) after the debug branch."""
    boxes = [fr['boxes'].copy() for fr in frames]
    poses = [[p.copy() for p in fr['poses']] for fr in frames]
    video_tracks, next_id = [], 0
    for f, fr in enumerate(frames):
        cur_boxes, cur_poses = boxes[f], poses[f]
        gt_boxes, gt_poses = fr['gt_boxes'], [el for el in fr['gt_kps']]
        if f == 0 and not ub:
            matches = -np.ones((cur_boxes.shape[0],), dtype=np.int32)
        elif ub:
            matches = compute_matches(gt_boxes, cur_boxes, gt_poses, cur_poses, w_iou, w_pck, algo)
        else:
            matches = compute_matches(boxes[f - 1], cur_boxes, poses[f - 1], cur_poses, w_iou, w_pck, algo)
        if ub:
            prev_tracks = np.asarray(fr['gt_tracks']).reshape(-1).tolist()
            kept = np.where(matches != -1)[0]
            matches = matches[kept]
            new_boxes = cur_boxes[kept]
            new_poses = [cur_poses[i] for i in kept]                     # references: _5 below writes through them
            if ub2:
                new_boxes[:, :4] = gt_boxes[matches]
                for k in range(matches.shape[0]):
                    rows = np.array(2) if conf_only else np.arange(3)
                    new_poses[k][rows, :] = fr['gt_kps'][matches[k]][rows, :]
            boxes[f], poses[f] = new_boxes, new_poses
        else:
            prev_tracks = video_tracks[f - 1] if f > 0 else None
        if ub5:
            mg = compute_matches(gt_boxes, cur_boxes, gt_poses, cur_poses, 1.0, 0.0, 'hungarian')
            for q in range(mg.shape[0]):
                if mg[q] != -1:
                    cur_poses[q][:3, :] = gt_poses[mg[q]][:3, :]
        tracks = []
        for m in matches:
            if m == -1:
                tracks.append(next_id)
                next_id += 1
                if next_id >= MAX_TRACK_IDS:
                    next_id %= MAX_TRACK_IDS
            else:
                tracks.append(prev_tracks[m])
        video_tracks.append(tracks)
    return boxes, poses, video_tracks


def _point(points, i):
    for q in points:
        if q['id'] is not None and q['id'][0] == i:
            return q
    return None


def mot_inputs_upper_bound(gtFrames, prFrames, distThresh=0.5):
    """motAll of assignGTmulti(..., computeUpperBound=True): in a frame with both GT and predictions only the predictions
    some GT selected (prToGT) stay, in ascending GT order, with the selecting GT's track id; frames without both reuse the
    last such frame's inputs."""
    J = ope.N_JOINTS
    motAll, mot = {}, None
    for f in range(len(gtFrames)):
        gts, prs = gtFrames[f]['annorect'], prFrames[f]['annorect']
        nG, nP = len(gts), len(prs)
        hasGT, gxy = np.zeros((nG, J), bool), np.zeros((nG, J, 2))
        tG = [r['track_id'][0] for r in gts]
        for g, r in enumerate(gts):
            pts = r['annopoints'][0]['point'] if len(r['annopoints']) > 0 else []
            for i in range(J):
                q = _point(pts, i)
                if q is not None:
                    hasGT[g, i] = True
                    gxy[g, i] = (q['x'][0], q['y'][0])
        hasPr, pxy = np.zeros((nP, J), bool), np.zeros((nP, J, 2))
        for p, r in enumerate(prs):
            for i in range(J):
                q = _point(r['annopoints'][0]['point'], i)
                if q is not None:
                    hasPr[p, i] = True
                    pxy[p, i] = (q['x'][0], q['y'][0])
        if nP and nG:
            dist = np.full((nP, nG, J), np.inf)
            for g, r in enumerate(gts):
                head = 0.6 * math.sqrt((r['x2'][0] - r['x1'][0]) * (r['x2'][0] - r['x1'][0]) +
                                       (r['y2'][0] - r['y1'][0]) * (r['y2'][0] - r['y1'][0]))
                dx = gxy[g, :, 0][None, :] - pxy[:, :, 0]
                dy = gxy[g, :, 1][None, :] - pxy[:, :, 1]
                with np.errstate(divide='ignore', invalid='ignore'):
                    d = np.sqrt(dx * dx + dy * dy) / head
                dist[:, g, :] = np.where(hasPr & hasGT[g][None, :], d, np.inf)
            nGTp = hasGT.sum(axis=1)
            match = dist <= distThresh
            pck = 1.0 * match.sum(axis=2)
            for j in range(nG):
                if nGTp[j] > 0:
                    pck[:, j] = pck[:, j] / nGTp[j]
            idx = np.argmax(pck, axis=1)
            for p in range(nP):
                keep = pck[p, idx[p]]
                pck[p, :] = 0
                pck[p, idx[p]] = keep
            prToGT = np.argmax(pck, axis=0)
            prToGT[np.max(pck, axis=0) == 0] = -1
            sel, sel_pos = prToGT[prToGT > -1], np.where(prToGT > -1)[0]       # :561-573
            dist, match, hasPr = dist[sel], match[sel], hasPr[sel]
            tP = [tG[g] for g in sel_pos]
            mot = {}
            for i in range(J):
                rg, rp = np.flatnonzero(hasGT[:, i]), np.flatnonzero(hasPr[:, i])
                dd = np.full((len(rg), len(rp)), np.nan)
                for a, g in enumerate(rg):
                    for b, p in enumerate(rp):
                        if match[p, g, i]:
                            dd[a, b] = dist[p, g, i]
                mot[i] = {'trackidxGT': [tG[g] for g in rg], 'trackidxPr': [tP[p] for p in rp], 'dist': dd}
        if mot is not None:
            motAll[f] = mot
    return motAll


def evaluate_tracking_upper_bound(gtFrames, prFrames):
    """evaluateTracking(..., trackUpperBound=True) -> (metrics [19, 1], per-sequence [(counts [15, 4], sumd [15])])."""
    motAll = mot_inputs_upper_bound(gtFrames, prFrames)
    per_seq = [ope.mot_sequence_counts(frames, motAll) for _, frames in ope.sequences(gtFrames)]
    return ope.mot_metrics([c for c, _ in per_seq], [d for _, d in per_seq]), per_seq
