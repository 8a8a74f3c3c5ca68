"""Device-tensor API over csrc/proposals.cu (RPN proposals, collect/distribute, box decode,
detection limit).  Tensors stay on the GPU; counts are device int32 (CUDA-graph friendly)."""
import ctypes as C

import numpy as np

from .. import _lib as L
from . import box_ops

BBOX_XFORM_CLIP = float(np.log(1000. / 16.))     # lib/core/config.py:672


def _nhwc_ld(t):
    """Leading dim of a [B,H,W,C'] tensor that may be a channel slice of a wider contiguous one."""
    B, H, W, _ = t.shape
    ld = t.stride(2)
    assert t.stride(3) == 1 and t.stride(1) == W * ld and (B == 1 or t.stride(0) == H * W * ld), \
        'expected an NHWC tensor (or a channel slice of one)'
    return ld


def rpn_proposals_levels(levels, im_info, pre_nms_topn, A, min_size=0.0, T=1, clip=BBOX_XFORM_CLIP, time_major=False):
    """All levels of a clip batch in ONE launch.  levels: list of dicts(logits, deltas, anchors, feat_stride,
    out [B, >=K, 4T+1] (may be a strided view), counts [B] (may be a strided view))."""
    torch = L.require_cuda()
    nl = len(levels)
    arr = (L.RpnLevel * nl)()
    Hs, Ws = (C.c_int * nl)(), (C.c_int * nl)()
    B = None
    out_bs = cnt_s = None
    for i, lv in enumerate(levels):
        lg, dl = lv['logits'], lv['deltas']
        assert lg.dtype == dl.dtype
        if time_major:
            Bq, Tt, H, W, _ = lg.shape
            assert Tt == T and dl.shape[:4] == lg.shape[:4]
            ld_s, ld_d = lg.stride(3), dl.stride(3)
            assert lg.stride(4) == 1 and dl.stride(4) == 1 and lg.stride(1) == H * W * ld_s
        else:
            Bq, H, W, _ = lg.shape
            ld_s, ld_d = _nhwc_ld(lg), _nhwc_ld(dl)
        B = Bq if B is None else B
        assert Bq == B and lv['anchors'].shape[0] == A
        o, c = lv['out'], lv['counts']
        assert o.dtype == torch.float32 and o.shape[-1] == 4 * T + 1 and o.stride(-1) == 1 and o.stride(-2) == 4 * T + 1
        if out_bs is None:
            out_bs, cnt_s = o.stride(0), c.stride(0)
        assert (o.stride(0) == out_bs and c.stride(0) == cnt_s) or B == 1
        arr[i] = L.RpnLevel(lg.data_ptr(), dl.data_ptr(), lv['anchors'].data_ptr(), ld_s, ld_d, H, W,
                            float(lv['feat_stride']), o.data_ptr(), c.data_ptr())
        Hs[i], Ws[i] = H, W
    act_f32 = int(levels[0]['logits'].dtype == torch.float32)
    need = C.c_size_t(0)
    L.call('dt_rpn_workspace_bytes', B, nl, Hs, Ws, A, C.byref(need))
    ws = box_ops._workspace(need.value, torch, slot='rpn')
    L.call('dt_rpn_proposals_multi', arr, nl, act_f32, B, A, T, L.ptr(im_info), int(pre_nms_topn), float(min_size), float(clip),
           out_bs, cnt_s, int(bool(time_major)), L.ptr(ws), ws.numel(), L.stream_ptr())


def rpn_proposals(logits, deltas, anchors, feat_stride, im_info, pre_nms_topn, min_size=0.0,
                  T=1, out=None, counts=None, clip=BBOX_XFORM_CLIP, time_major=False):
    """One level.  logits [B,H,W,A], deltas [B,H,W,4AT] (fp32 or bf16; channel slices of a wider NHWC tensor
    are fine; [B,T,H,W,.] when time_major), anchors [A,4T] fp64 cuda, im_info [B,3] fp32 cuda.
    Returns (props [B,K,4T+1] fp32, counts [B] int32)."""
    torch = L.require_cuda()
    B = logits.shape[0]
    H, W = (logits.shape[2], logits.shape[3]) if time_major else (logits.shape[1], logits.shape[2])
    A = anchors.shape[0]
    n = H * W * A
    K = n if (pre_nms_topn <= 0 or pre_nms_topn > n) else pre_nms_topn
    if out is None:
        out = L.zeros((B, K, 4 * T + 1), torch.float32)
    if counts is None:
        counts = L.zeros((B,), torch.int32)
    assert out.shape[-2] >= K
    rpn_proposals_levels([dict(logits=logits, deltas=deltas, anchors=anchors, feat_stride=feat_stride, out=out, counts=counts)],
                         im_info, pre_nms_topn, A, min_size, T, clip, time_major)
    return out, counts


def collect(props, keep, nkeep, post_nms_topn, R=None):
    """props [B,L,K,4T+1], keep [B*L,K], nkeep [B*L] -> rois [B,R,4T+1], scores [B,R], counts [B]."""
    torch = L.require_cuda()
    B, Lv, K, ld = props.shape
    T = (ld - 1) // 4
    R = R or (post_nms_topn if post_nms_topn > 0 else Lv * K)
    rois = L.zeros((B, R, ld), torch.float32)
    scores = L.zeros((B, R), torch.float32)
    counts = L.zeros((B,), torch.int32)
    L.call('dt_collect_rpn', L.ptr(props.contiguous()), L.ptr(keep.contiguous()), L.ptr(nkeep.contiguous()), B, Lv, K, T,
           int(post_nms_topn), L.ptr(rois), L.ptr(scores), L.ptr(counts), R, L.stream_ptr())
    return rois, scores, counts


def distribute(rois, n_dev=None, col0=1, T=1, k_min=2, k_max=5, s0=224.0, lvl0=4.0, want_restore=True):
    """rois [n, ld] -> (levels [n] int32, idx_restore [n] int32 or None, level_counts)."""
    torch = L.require_cuda()
    rois = rois.contiguous()
    n, ld = rois.shape
    levels = L.zeros((max(n, 1),), torch.int32)
    restore = L.zeros((max(n, 1),), torch.int32) if want_restore else None
    lc = L.zeros((k_max - k_min + 1,), torch.int32)
    L.call('dt_distribute_fpn', L.ptr(rois), n, L.ptr(n_dev), ld, col0, T, k_min, k_max, float(s0), float(lvl0),
           L.ptr(levels), L.ptr(restore), L.ptr(lc), L.stream_ptr())
    return levels[:n], (restore[:n] if want_restore else None), lc


def box_decode(rois, roi_counts, cls_logits, bbox_deltas, num_classes, im_info, im_hw,
               weights=(10., 10., 5., 5.), score_thresh=0.05, T=1, clip=BBOX_XFORM_CLIP):
    """rois [B,R,4T+1]; cls_logits [B*R, >=C]; bbox_deltas [B*R, >=4TC] fp32.
    Returns dets [B, C-1, R, 4T+1], det_counts [B*(C-1)]."""
    torch = L.require_cuda()
    B, R, _ = rois.shape
    dets = L.zeros((B, num_classes - 1, R, 4 * T + 1), torch.float32)
    cnt = L.zeros((B * (num_classes - 1),), torch.int32)
    w4 = (C.c_float * 4)(*[float(w) for w in weights])
    assert cls_logits.dtype == torch.float32 and bbox_deltas.dtype == torch.float32
    assert cls_logits.stride(1) == 1 and bbox_deltas.stride(1) == 1
    L.call('dt_box_decode', L.ptr(rois.contiguous()), L.ptr(roi_counts), B, R, T, C.c_void_p(cls_logits.data_ptr()),
           cls_logits.stride(0), C.c_void_p(bbox_deltas.data_ptr()), bbox_deltas.stride(0), num_classes, L.ptr(im_info), L.ptr(im_hw), w4, float(clip),
           float(score_thresh), L.ptr(dets), L.ptr(cnt), L.stream_ptr())
    return dets, cnt


def limit_detections(dets, keep, nkeep, max_per_im, cap=None):
    """dets [B,C-1,R,ld], keep [B*(C-1), R], nkeep -> out [B, C-1, cap, ld], counts [B*(C-1)]."""
    torch = L.require_cuda()
    B, C1, R, ld = dets.shape
    T = (ld - 1) // 4
    cap = cap or R
    out = L.zeros((B, C1, cap, ld), torch.float32)
    cnt = L.zeros((B * C1,), torch.int32)
    L.call('dt_limit_detections', L.ptr(dets), L.ptr(keep.contiguous()), L.ptr(nkeep), B, C1 + 1, R, T, int(max_per_im),
           L.ptr(out), L.ptr(cnt), cap, L.stream_ptr())
    return out, cnt


def generate_proposals_level(logits, deltas, anchors, feat_stride, im_info, pre_nms_topn, post_nms_topn,
                             nms_thresh, min_size=0.0, T=1):
    """Full GenerateProposalsOp for one level (generate_proposals.py:40-181): returns
    (props [B,K,4T+1], keep [B,K], nkeep [B]) — rois = props[b, keep[b, :nkeep[b]]]."""
    props, counts = rpn_proposals(logits, deltas, anchors, feat_stride, im_info, pre_nms_topn, min_size, T)
    cmp_mode = box_ops.NMS_2D_GE if T == 1 else box_ops.NMS_TUBE_GT
    order = box_ops.ORDER_INDEX if T == 1 else box_ops.ORDER_SCORE
    keep, nkeep = box_ops.nms_batched(props, counts, nms_thresh, cmp_mode, order, max_keep=post_nms_topn)
    return props, keep, nkeep


def aug_merge_dets(dets, counts, flips, im_hw):
    """Test-time augmentation union (lib/core/test.py:338-414, UNION heuristics): V views' box_decode outputs
    (dets [B, C-1, R, 5], counts [B*(C-1)]) stacked per (image, class) in view order, a view with flips[v] flipped back
    with the image width im_hw[b, 1].  Returns (union [B, C-1, V*R, 5], counts [B*(C-1)]), nms_batched's layout."""
    torch = L.require_cuda()
    V = len(dets)
    assert V == len(counts) == len(flips) and V >= 1
    B, C1, R, ld = dets[0].shape
    assert ld == 5 and all(d.shape == dets[0].shape and d.dtype == torch.float32 and d.is_contiguous() for d in dets)
    assert im_hw.dtype == torch.float32 and im_hw.shape == (B, 2) and im_hw.is_contiguous()
    out = L.zeros((B, C1, V * R, 5), torch.float32)
    cnt = L.zeros((B * C1,), torch.int32)
    L.call('dt_aug_merge_dets', (C.c_void_p * V)(*[d.data_ptr() for d in dets]),
           (C.c_void_p * V)(*[c.data_ptr() for c in counts]), (C.c_int * V)(*[int(bool(f)) for f in flips]), V, B, C1 + 1, R,
           C.c_void_p(im_hw.data_ptr() + 4), 2, L.ptr(out), L.ptr(cnt), L.stream_ptr())
    return out, cnt
