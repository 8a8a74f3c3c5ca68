"""Oracle: soft-NMS and bounding-box voting (TEST INFRASTRUCTURE ONLY).

Restates, vectorised per round / per row in numpy:
  lib/utils/cython_nms.pyx:98-203 soft_nms   in the C that Cython emits for it: the '+ 1' is the C double 1.0, so
      widths and areas are fp64 products rounded to fp32 where stored (area, iw, ih, ua); iw*ih, ov and the decayed
      score are fp32; the gaussian weight is np.exp of an fp32 argument in fp64, stored fp32.  The pick is the first
      maximum from position i (strict <), swapped with row i; a row that overlaps the pick and decays below
      `threshold` is replaced by the current last row, which is then decayed at its new position.  Within a round
      every row is decayed once, so the k-th discarded position below the new N receives the k-th largest surviving
      position at or above it.
  lib/core/test.py:750-806 box_results_with_nms_and_limit with TEST.SOFT_NMS / TEST.BBOX_VOTE (the rows of the
      reference's (dets, inds) soft_nms tuple taken as Detectron does, DESIGN.md §4).
  lib/utils/boxes.py:294-310 box_voting     np.average(boxes, axis=0, weights=scores) under numpy 2.x in fp32: a
      sequential sum of box * w over the matched rows (a reduction over the outer axis), numpy's pairwise_sum of the
      weights, one division.
Checked bit for bit against the compiled reference (tests/golden/soft_nms.npz, tests/test_soft_nms.py)."""
import numpy as np

from . import boxes as obox
from .boxes import bbox_overlaps_2d

F32, F64 = np.float32, np.float64
METHODS = {'hard': 0, 'linear': 1, 'gaussian': 2}


def _cy_min(a, b):
    return np.where(a <= b, a, b)


def _cy_max(a, b):
    return np.where(a >= b, a, b)


def soft_nms(dets, sigma=0.5, Nt=0.3, threshold=0.001, method=0):
    """cython_nms.soft_nms(boxes_in, sigma, Nt, threshold, method) -> (rows [N, 5] fp32, inds [N] int64)."""
    boxes = np.array(dets, dtype=F32)[:, :5]
    sigma, Nt, threshold = F32(sigma), F32(Nt), F32(threshold)
    n = boxes.shape[0]
    rows = np.arange(n)                      # source row at each position
    sc = boxes[:, 4].copy()                  # score at each position
    x1, y1, x2, y2 = (boxes[:, c] for c in range(4))
    N, i = n, 0
    while i < N:
        seg = sc[i:N].copy()
        if not np.isnan(seg[0]):
            seg[np.isnan(seg)] = -np.inf     # no comparison with NaN succeeds
            m = i + int(np.argmax(seg))      # first maximum
        else:
            m = i
        rows[[i, m]], sc[[i, m]] = rows[[m, i]], sc[[m, i]]
        t = rows[i]
        tx1, ty1, tx2, ty2 = x1[t], y1[t], x2[t], y2[t]
        r = rows[i + 1:N]
        s = sc[i + 1:N]
        area = (((x2[r] - x1[r]).astype(F64) + 1.0) * ((y2[r] - y1[r]).astype(F64) + 1.0)).astype(F32)
        iw = ((_cy_min(tx2, x2[r]) - _cy_max(tx1, x1[r])).astype(F64) + 1.0).astype(F32)
        ih = ((_cy_min(ty2, y2[r]) - _cy_max(ty1, y1[r])).astype(F64) + 1.0).astype(F32)
        ok = (iw > 0) & (ih > 0)
        inter = iw * ih
        at = (F64(tx2 - tx1) + 1.0) * (F64(ty2 - ty1) + 1.0)
        with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
            ua = ((at + area.astype(F64)) - inter.astype(F64)).astype(F32)
            ov = inter / ua
            if method == 1:
                w = np.where(ov > Nt, (1.0 - ov.astype(F64)).astype(F32), F32(1))
            elif method == 2:
                w = np.exp((-(ov * ov) / sigma).astype(F64)).astype(F32)
            else:
                w = np.where(ov > Nt, F32(0), F32(1))
            new = np.where(ok, (w * s).astype(F32), s)
            disc = ok & (new < threshold)
        sc[i + 1:N] = new
        D = int(disc.sum())
        if D:
            newN = N - D
            pos = np.arange(i + 1, N)
            holes = pos[disc & (pos < newN)]
            donors = pos[~disc & (pos >= newN)][::-1]
            rows[holes], sc[holes] = rows[donors], sc[donors]
            N = newN
        i += 1
    out = np.concatenate([boxes[rows[:N], :4], sc[:N, None]], axis=1).astype(F32)
    return out, rows[:N].astype(np.int64)


_soft_nms = soft_nms        # box_results_with_nms_and_limit's `soft_nms` keyword shadows the name


def pairwise_sum(x):
    """numpy's pairwise_sum (umath loops) of an fp32 vector, in fp32."""
    x = np.asarray(x, dtype=F32)
    n = len(x)
    if n < 8:
        r = F32(0)
        for v in x:
            r = F32(r + v)
        return r
    if n <= 128:
        m = n - n % 8
        a = np.cumsum(x[:m].reshape(-1, 8), axis=0, dtype=F32)[-1]
        r = F32(F32(F32(a[0] + a[1]) + F32(a[2] + a[3])) + F32(F32(a[4] + a[5]) + F32(a[6] + a[7])))
        for v in x[m:]:
            r = F32(r + v)
        return r
    n2 = n // 2
    n2 -= n2 % 8
    return F32(pairwise_sum(x[:n2]) + pairwise_sum(x[n2:]))


def weighted_average(boxes, w):
    """np.average(boxes [n, 4] fp32, axis=0, weights=w [n] fp32) as numpy 2.x evaluates it."""
    num = np.cumsum((boxes * w[:, None]).astype(F32), axis=0, dtype=F32)[-1]
    return (num / pairwise_sum(w)).astype(F32)


def box_voting(top_dets, all_dets, thresh):
    """boxes.py:294-310 box_voting(top_dets, all_dets, thresh) for 2-D rows [n, 5]."""
    top = np.asarray(top_dets, dtype=F32)
    alld = np.asarray(all_dets, dtype=F32)
    out = top.copy()
    if top.shape[0] == 0:
        return out
    ov = bbox_overlaps_2d(top[:, :4], alld[:, :4])
    for k in range(top.shape[0]):
        idx = np.where(ov[k] >= thresh)[0]
        out[k, :4] = weighted_average(alld[idx, :4], alld[idx, 4])
    return out


def box_results_with_nms_and_limit(scores, boxes, num_classes=2, score_thresh=0.05, nms_thresh=0.5, dets_per_im=100,
                                   soft_nms=None, bbox_vote=None):
    """test.py:750-806 with its two options: soft_nms None (hard NMS) or (method name, sigma) of TEST.SOFT_NMS
    (score_thresh 0.0001, as :777-782 passes it); bbox_vote None or TEST.BBOX_VOTE.VOTE_TH.  With both None this is
    oracle/detections.box_results_with_nms_and_limit."""
    T = boxes.shape[-1] // (num_classes * 4)
    cls_boxes = [[] for _ in range(num_classes)]
    for j in range(1, num_classes):
        inds = np.where(scores[:, j] > F32(score_thresh))[0]
        dets_j = np.hstack((boxes[inds, j * 4 * T:(j + 1) * 4 * T], scores[inds, j][:, None])).astype(F32, copy=False)
        if soft_nms is not None:
            method, sigma = soft_nms
            nms_dets = _soft_nms(dets_j, sigma, nms_thresh, 0.0001, METHODS[method])[0]
        else:
            keep = obox.nms(dets_j, nms_thresh)
            nms_dets = dets_j[np.asarray(keep, dtype=np.int64), :] if len(keep) else dets_j[:0]
        if bbox_vote is not None:
            nms_dets = box_voting(nms_dets, dets_j, bbox_vote)
        cls_boxes[j] = nms_dets
    if dets_per_im > 0:
        image_scores = np.hstack([cls_boxes[j][:, -1] for j in range(1, num_classes)])
        if len(image_scores) > dets_per_im:
            th = np.sort(image_scores)[-dets_per_im]
            for j in range(1, num_classes):
                cls_boxes[j] = cls_boxes[j][np.where(cls_boxes[j][:, -1] >= th)[0], :]
    im_results = np.vstack([cls_boxes[j] for j in range(1, num_classes)])
    return im_results[:, -1], im_results[:, :-1], cls_boxes
