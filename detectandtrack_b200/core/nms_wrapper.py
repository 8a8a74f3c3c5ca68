"""Drop-in for lib/core/nms_wrapper.py: ``nms(dets, thresh)`` / ``tube_nms`` / ``soft_nms``.
Same dispatch (5 columns -> 2-D '>=' NMS returning ascending indices; more ->
tube NMS returning a score-ordered list), computed by csrc/boxes.cu."""
import numpy as np

from .. import _lib as L
from ..ops import box_ops


def _run(dets, thresh, cmp_mode, out_order):
    import torch
    d = torch.from_numpy(np.ascontiguousarray(dets, dtype=np.float32)).cuda().unsqueeze(0)
    keep, num = box_ops.nms_batched(d, None, thresh, cmp_mode, out_order)
    n = int(num[0].item())
    return keep[0, :n].cpu().numpy().astype(np.int64)


def soft_nms(dets, sigma=0.5, overlap_thresh=0.3, score_thresh=0.001, method='linear'):
    """lib/core/nms_wrapper.py:29-46: (rows [n, 5] fp32, inds [n] int64) as cython_nms.soft_nms returns them, or
    `dets` itself when it is empty."""
    if dets.shape[0] == 0:
        return dets
    if dets.shape[1] > 5:
        raise NotImplementedError('Need to handle tubes..')
    assert method in L.SOFT_NMS_METHODS, 'Unknown soft_nms method: {}'.format(method)
    import torch
    d = torch.from_numpy(np.ascontiguousarray(dets, dtype=np.float32)).cuda().unsqueeze(0)
    rows, inds, num = box_ops.soft_nms_batched(d, None, np.float32(sigma), np.float32(overlap_thresh),
                                               np.float32(score_thresh), method)
    n = int(num[0].item())
    return rows[0, :n].cpu().numpy(), inds[0, :n].cpu().numpy().astype(np.int64)


def nms(dets, thresh, soft_nms=False):
    """lib/core/nms_wrapper.py:49-57."""
    if soft_nms:
        raise NotImplementedError('soft-NMS is not on the hot path (nms_wrapper.py:29-46)')
    if dets.shape[0] == 0:
        return []
    if dets.shape[1] > 5:
        return tube_nms(dets, thresh)
    return _run(dets, thresh, box_ops.NMS_2D_GE, box_ops.ORDER_INDEX)


def tube_nms(dets, thresh):
    """lib/core/nms_wrapper.py:60-70 -> lib/nms/py_cpu_nms_tubes.py:17-53."""
    if (dets.shape[1] - 1) % 4 != 0:
        raise RuntimeError('tube_nms: expected N x (4*T+1) dets, got %s' % (dets.shape,))
    return _run(dets, thresh, box_ops.NMS_TUBE_GT, box_ops.ORDER_SCORE).tolist()
