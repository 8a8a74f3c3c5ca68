"""Device-tensor API over csrc/targets.cu: the training target generators (lib/roi_data/rpn.py, fast_rcnn.py,
keypoint_rcnn.py; lib/datasets/json_dataset.py add_proposals) on the device.  See include/dt_b200.h."""
import ctypes as C

from .. import _lib as L
from . import box_ops

M64 = (1 << 64) - 1
SCALE_STREAM = 5          # stream of the training-scale draw (streams 0..4 are csrc/targets.cu's)


def hash_u32(seed, stream, image, i):
    """csrc/targets.cu's counter-based generator on the host: splitmix64 finaliser over seed, stream, image and index
    (unsigned 64-bit wrap-around) -> the high 32 bits."""
    x = (seed * 0x9E3779B97F4A7C15 + stream * 0xBF58476D1CE4E5B9 + image * 0x94D049BB133111EB + i) & M64
    x ^= x >> 30
    x = (x * 0xBF58476D1CE4E5B9) & M64
    x ^= x >> 27
    x = (x * 0x94D049BB133111EB) & M64
    x ^= x >> 31
    return x >> 32


def train_scale(scales, seed, n):
    """The TRAIN.SCALES entry of the n-th clip of a run (n = it * world * B + rank * B + j): randint(len(SCALES)) on
    stream 5, the reference's per-image npr.randint draw (minibatch.py:73-74) as a pure function of (seed, n)."""
    return scales[(hash_u32(int(seed), SCALE_STREAM, 0, int(n)) * len(scales)) >> 32]


def rpn_targets(level_shapes, anchors, strides, A, gt_boxes, gt_counts, im_info, cfg_train, seed, gt_visible=None):
    """level_shapes: [(H, W)] finest first; anchors: per level [A, 4T] fp64 device cell anchors; gt_boxes [B, Gmax, 4T] fp32
    (original image coordinates, non-crowd; T = 1 boxes or T <= 4 frame tubes), gt_visible [B, Gmax, T] uint8 or None,
    gt_counts [B] int32, im_info [B, 3].  Returns per level dict(labels [B,H,W,A] i32, bbox_targets / inside / outside
    [B,H,W,4T*A] f32, vis_labels [B,H,W,T*A] i32) (rpn.py:206-381)."""
    torch = L.require_cuda()
    B, Gmax, D = gt_boxes.shape
    T = D // 4
    nl = len(level_shapes)
    arr = (L.RpnTargetLevel * nl)()
    Hs, Ws = (C.c_int * nl)(), (C.c_int * nl)()
    out = []
    for i, (H, W) in enumerate(level_shapes):
        o = dict(labels=torch.empty((B, H, W, A), dtype=torch.int32, device='cuda'),
                 bbox_targets=torch.empty((B, H, W, 4 * T * A), dtype=torch.float32, device='cuda'),
                 inside=torch.empty((B, H, W, 4 * T * A), dtype=torch.float32, device='cuda'),
                 outside=torch.empty((B, H, W, 4 * T * A), dtype=torch.float32, device='cuda'),
                 vis_labels=torch.empty((B, H, W, T * A), dtype=torch.int32, device='cuda'))
        out.append(o)
        a = anchors[i]
        assert a.dtype == torch.float64 and tuple(a.shape) == (A, 4 * T) and a.is_contiguous()
        arr[i] = L.RpnTargetLevel(H, W, float(strides[i]), a.data_ptr(), o['labels'].data_ptr(), o['bbox_targets'].data_ptr(),
                                  o['inside'].data_ptr(), o['outside'].data_ptr(), o['vis_labels'].data_ptr())
        Hs[i], Ws[i] = H, W
    need = C.c_size_t(0)
    L.call('dt_rpn_targets_workspace_bytes', B, nl, Hs, Ws, A, Gmax, C.byref(need))
    ws = box_ops._workspace(need.value, torch, slot='rpn_targets')
    assert gt_boxes.dtype == torch.float32 and gt_counts.dtype == torch.int32 and im_info.dtype == torch.float32
    assert gt_visible is None or (gt_visible.dtype == torch.uint8 and tuple(gt_visible.shape) == (B, Gmax, T))
    L.call('dt_rpn_targets', arr, nl, A, T, B, L.ptr(gt_boxes), L.ptr(gt_visible), L.ptr(gt_counts), Gmax, L.ptr(im_info),
           float(cfg_train.RPN_STRADDLE_THRESH), float(cfg_train.RPN_POSITIVE_OVERLAP), float(cfg_train.RPN_NEGATIVE_OVERLAP),
           int(cfg_train.RPN_BATCH_SIZE_PER_IM), float(cfg_train.RPN_FG_FRACTION), int(seed), L.ptr(ws), ws.numel(), L.stream_ptr())
    return out


def sample_rois(rois, roi_scores, roi_counts, gt, im_info, cfg, seed, keypoints=True, totals=None):
    """rois [B, R, 5] / roi_scores [B, R] / roi_counts [B]: rpn_ops.collect's per-image output.  gt: dict(boxes [B,Gmax,4] f32,
    classes / crowd [B,Gmax] i32, keypoints [B,Gmax,3,K] i32, counts [B] i32).  Returns the Fast R-CNN / keypoint blobs as
    fixed-capacity device tensors (see dt_sample_rois)."""
    torch = L.require_cuda()
    B, R, ldr = rois.shape
    T = (ldr - 1) // 4
    assert gt['boxes'].shape[2] == 4 * T, 'gt boxes must be [B, Gmax, 4T] like the rois'
    Gmax = gt['boxes'].shape[1]
    tr = cfg.TRAIN
    batch = int(tr.BATCH_SIZE_PER_IM)
    nc = int(cfg.MODEL.NUM_CLASSES)
    K = int(cfg.KRCNN.NUM_KEYPOINTS) if keypoints else 0
    fg_per = int(round(tr.FG_FRACTION * batch))
    kcap = (max(fg_per, Gmax) + 7) // 8 * 8
    f32, i32 = torch.float32, torch.int32
    o = dict(rois=torch.empty((B, batch, 4 * T + 1), dtype=f32, device='cuda'), labels=torch.empty((B, batch), dtype=i32, device='cuda'),
             bbox_targets=torch.empty((B, batch, 4 * T * nc), dtype=f32, device='cuda'),
             inside=torch.empty((B, batch, 4 * T * nc), dtype=f32, device='cuda'),
             outside=torch.empty((B, batch, 4 * T * nc), dtype=f32, device='cuda'), counts=torch.empty((B,), dtype=i32, device='cuda'),
             totals=totals if totals is not None else L.zeros((2,), f32))
    if keypoints:
        assert gt['keypoints'].shape[3] == K * T, 'gt keypoints must be [B, Gmax, 3, K*T]'
        o.update(kp_rois=torch.empty((B, kcap, 4 * T + 1), dtype=f32, device='cuda'), kp_locations=torch.empty((B, kcap, K * T), dtype=i32, device='cuda'),
                 kp_weights=torch.empty((B, kcap, K * T), dtype=f32, device='cuda'), kp_counts=torch.empty((B,), dtype=i32, device='cuda'))
    w4 = (C.c_float * 4)(*[float(x) for x in cfg.MODEL.BBOX_REG_WEIGHTS])
    L.call('dt_sample_rois', L.ptr(rois), L.ptr(roi_scores), L.ptr(roi_counts), B, R, int(tr.RPN_POST_NMS_TOP_N),
           L.ptr(gt['boxes']), L.ptr(gt['classes']), L.ptr(gt['crowd']), L.ptr(gt.get('keypoints') if keypoints else None),
           L.ptr(gt['counts']), Gmax, K, T, L.ptr(im_info), nc, batch, float(tr.FG_FRACTION), float(tr.FG_THRESH),
           float(tr.BG_THRESH_HI), float(tr.BG_THRESH_LO), w4, int(cfg.KRCNN.HEATMAP_SIZE) if keypoints else 0, int(seed),
           L.ptr(o['rois']), L.ptr(o['labels']), L.ptr(o['bbox_targets']), L.ptr(o['inside']), L.ptr(o['outside']), L.ptr(o['counts']),
           L.ptr(o.get('kp_rois')), L.ptr(o.get('kp_locations')), L.ptr(o.get('kp_weights')), L.ptr(o.get('kp_counts')), kcap,
           L.ptr(o['totals']), L.stream_ptr())
    return o
