"""Host mirror of the lib/utils/boxes.py entry points that sit on the hot path.
Tube-aware IoU runs on the device; the tiny layout helpers stay numpy."""
import numpy as np

from ..ops import box_ops


def _strip_score(a):
    a = np.asarray(a)
    if a.shape[1] % 4 == 0:
        return a
    if (a.shape[1] - 1) % 4 == 0:
        return a[:, :-1]
    raise ValueError('Invalid tube dimensions {}'.format(a.shape))


def bbox_overlaps(boxes, query_boxes):
    """lib/utils/boxes.py:60-69: mean-over-frames IoU of (N,4T[+1]) vs (K,4T[+1])."""
    import torch
    b = np.ascontiguousarray(_strip_score(boxes), dtype=np.float32)
    q = np.ascontiguousarray(_strip_score(query_boxes), dtype=np.float32)
    T = b.shape[1] // 4
    if q.shape[1] // 4 != T:
        raise RuntimeError('bbox_overlaps: tube lengths differ: %s vs %s' % (b.shape, q.shape))
    return box_ops.bbox_overlaps(torch.from_numpy(b).cuda(), torch.from_numpy(q).cuda(), T=T).cpu().numpy()


def box_voting(top_dets, all_dets, thresh):
    """lib/utils/boxes.py:294-310: each row of top_dets [N, 5] with its box replaced by the score-weighted average of
    the all_dets [M, 5] boxes whose IoU with it is >= thresh (computed on the device)."""
    import torch
    top = np.asarray(top_dets)
    if top.shape[1] != 5 or np.asarray(all_dets).shape[1] != 5:
        raise NotImplementedError('box_voting: 2-D boxes [N, 5] only, got %s / %s' % (top.shape, np.asarray(all_dets).shape))
    out = top.copy()
    if top.shape[0] == 0:
        return out
    a = torch.from_numpy(np.ascontiguousarray(all_dets, dtype=np.float32)).cuda().unsqueeze(0)
    t = torch.from_numpy(np.ascontiguousarray(top, dtype=np.float32)).cuda().unsqueeze(0)
    n = torch.tensor([top.shape[0]], dtype=torch.int32, device='cuda')
    rows, _ = box_ops.box_vote(a, None, thresh, top=t, top_counts=n)
    out[:, :4] = rows[0, :top.shape[0], :4].cpu().numpy()
    return out


def boxes_area(boxes):
    """lib/utils/boxes.py:72-78."""
    w = (boxes[:, 2::4] - boxes[:, 0::4] + 1)
    h = (boxes[:, 3::4] - boxes[:, 1::4] + 1)
    areas = np.mean(w * h, axis=1)
    assert np.all(areas >= 0), 'Negative areas founds'
    return areas


def flip_boxes(boxes, im_width):
    """lib/utils/boxes.py:275-282 for boxes or T-frame tubes [n, 4T]: x1' = width - x2 - 1, x2' = width - x1 - 1 in every
    frame's columns (0::4 and 2::4)."""
    boxes = np.asarray(boxes)
    flipped = boxes.copy()
    flipped[:, 0::4] = im_width - boxes[:, 2::4] - 1
    flipped[:, 2::4] = im_width - boxes[:, 0::4] - 1
    assert np.all(flipped[:, 2::4] >= flipped[:, 0::4])
    return flipped
