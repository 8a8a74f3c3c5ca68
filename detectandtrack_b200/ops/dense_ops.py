"""Device-tensor API over csrc/dense_ops.cu (image prep, max-pool, RoIAlign, keypoint decode)."""
import ctypes as C

from .. import _lib as L


def prep_clip(frames_u8, pixel_means, im_scale, out_hw, pad_hw, cpad=8, out_f32=False, border=(0, 0), row_planes=False):
    """frames [F,H,W,3] uint8 cuda (BGR) -> [F,Hp+2by,Wp+2bx,cpad] (pixel - mean), resized, zero padded,
    with `border` = (by, bx) physical zero rows / pixels on every side.  row_planes: the padded rows are
    de-interleaved by parity, [F, 2, (Hp+2by)/2, Wp+2bx, cpad] (the layout conv1_7x7s2 reads)."""
    torch = L.require_cuda()
    F, H, W, _ = frames_u8.shape
    Hr, Wr = out_hw
    Hp, Wp = pad_hw
    by, bx = border
    Ht, Wt = Hp + 2 * by, Wp + 2 * bx
    # out_f32: False/0 bf16, True/1 fp32 rounded to tf32, 2 raw fp32, 3 bf16 split pixel [hi3 | lo3 | 0 0] (cpad 8)
    shape = (F, 2, Ht // 2, Wt, cpad) if row_planes else (F, Ht, Wt, cpad)
    out = torch.empty(shape, dtype=torch.float32 if out_f32 in (True, 1, 2) else torch.bfloat16, device='cuda')
    m = (C.c_float * 3)(*[float(v) for v in pixel_means])
    L.call('dt_prep_clip', L.ptr(frames_u8.contiguous()), F, H, W, m, float(im_scale), Hr, Wr, Hp, Wp, cpad, by, bx,
           int(bool(row_planes)), int(out_f32), L.ptr(out), L.stream_ptr())
    return out


def prep_batch(clips, pixel_means, im_scales, out_hws, flips, pad_hw, cpad=8, out_f32=False, border=(0, 0), row_planes=False):
    """clips: B uint8 cuda tensors [T, H_b, W_b, 3] (BGR; sizes may differ), each resized by im_scales[b] to out_hws[b],
    its source mirrored horizontally first where flips[b] -> [B*T, ...] in prep_clip's layout at the shared pad_hw.
    With flips[b] == 0, clip b's slice equals prep_clip of that clip byte for byte."""
    torch = L.require_cuda()
    B = len(clips)
    T = clips[0].shape[0] if B else 0
    assert all(c.dtype == torch.uint8 and c.dim() == 4 and c.shape[0] == T and c.shape[3] == 3 and c.is_contiguous() for c in clips)
    Hp, Wp = pad_hw
    by, bx = border
    Ht, Wt = Hp + 2 * by, Wp + 2 * bx
    shape = (B * T, 2, Ht // 2, Wt, cpad) if row_planes else (B * T, Ht, Wt, cpad)
    out = torch.empty(shape, dtype=torch.float32 if out_f32 in (True, 1, 2) else torch.bfloat16, device='cuda')
    ints = lambda v: (C.c_int * B)(*[int(x) for x in v])
    L.call('dt_prep_batch', (C.c_void_p * B)(*[c.data_ptr() for c in clips]), ints([c.shape[1] for c in clips]),
           ints([c.shape[2] for c in clips]), (C.c_double * B)(*[float(s) for s in im_scales]), ints([h for h, _ in out_hws]),
           ints([w for _, w in out_hws]), ints([bool(f) for f in flips]), B, T, (C.c_float * 3)(*[float(v) for v in pixel_means]),
           Hp, Wp, cpad, by, bx, int(bool(row_planes)), int(out_f32), L.ptr(out), L.stream_ptr())
    return out


def maxpool2d(x, k, s, p, x3=False):
    """x [N,H,W,C] -> [N,Ho,Wo,C] (floor mode).  x3: rows are [hi | lo] tf32 pairs (C = row / 2)."""
    torch = L.require_cuda()
    N, H, W, ld = x.shape
    Cc = ld // 2 if x3 else ld
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    y = torch.empty((N, Ho, Wo, ld), dtype=x.dtype, device='cuda')
    L.call('dt_maxpool2d', L.ptr(x), N, H, W, Cc, ld, k, s, p, int(x.dtype == torch.float32), int(bool(x3)), L.ptr(y), ld,
           L.stream_ptr())
    return y


def roi_align(feats, scales, rois, levels, P, sampling_ratio, T=1, k_min=2, n_dev=None, channels=None,
              round_tf32=False, x3_mode=0):
    """feats: list of [Nimg*T, H_l, W_l, C] (finest first, level k_min + i); rois [R, 4T+1] fp32
    (col 0 = image index); levels [R] int32 or None for a single level -> [R, T, P, P, C]."""
    torch = L.require_cuda()
    nl = len(feats)
    ldf = feats[0].shape[-1]
    Cc = channels or (ldf // 2 if x3_mode else ldf)
    R = rois.shape[0]
    # x3_mode 1: [R,T,P,P,2C] per-position [hi | lo]; 2: [R, 2*T*P*P*C] planar hi block | lo block
    oshape = (R, T, P, P, 2 * Cc) if x3_mode == 1 else ((R, 2 * T * P * P * Cc) if x3_mode == 2 else (R, T, P, P, Cc))
    out = torch.empty(oshape, dtype=feats[0].dtype, device='cuda')
    fp = (C.c_void_p * nl)(*[f.data_ptr() for f in feats])
    Hs = (C.c_int * nl)(*[f.shape[1] for f in feats])
    Ws = (C.c_int * nl)(*[f.shape[2] for f in feats])
    sc = (C.c_float * nl)(*[float(s) for s in scales])
    for f in feats:
        assert f.is_contiguous() and f.dtype == feats[0].dtype and f.shape[-1] == ldf
    rois = rois.contiguous()
    L.call('dt_roi_align', fp, Hs, Ws, sc, nl, k_min, Cc, ldf, int(feats[0].dtype == torch.float32), L.ptr(rois),
           rois.shape[1], L.ptr(n_dev), R, T, L.ptr(levels), P, sampling_ratio, int(bool(round_tf32)), int(x3_mode),
           L.ptr(out), L.stream_ptr())
    return out


def keypoint_decode(lowres, boxes, K=17, T=1, n_dev=None, min_size=0, want_heatmaps=False):
    """lowres [D*T, S, S, >=4K] fp32 (sub-pixel packed), boxes [D, >=4T] image space.
    Returns (xy_preds [D,4,T*K], heatmaps [D,T*K,4S,4S] or None)."""
    torch = L.require_cuda()
    DT_, S, _, ldl = lowres.shape
    D = DT_ // T
    xy = L.zeros((D, 4, T * K), torch.float32)
    heat = L.zeros((D, T * K, 4 * S, 4 * S), torch.float32) if want_heatmaps else None
    assert boxes.stride(1) == 1 and boxes.dtype == torch.float32
    assert lowres.dtype == torch.float32 and lowres.is_contiguous()
    L.call('dt_keypoint_decode', L.ptr(lowres), ldl, S, K, T, C.c_void_p(boxes.data_ptr()), boxes.stride(0), L.ptr(n_dev), D, int(min_size),
           L.ptr(heat), L.ptr(xy), L.stream_ptr())
    return xy, heat


def scale_rois(boxes, ncols, im_scale, batch_idx=None, per_image=1):
    """boxes [n, >=ncols] fp32 (row stride free) -> rois [n, ncols+1] = (image index, boxes * im_scale in fp64 -> fp32)
    (lib/core/test.py:76-113); image index = batch_idx[i] or i // per_image."""
    torch = L.require_cuda()
    n = boxes.shape[0]
    assert boxes.dtype == torch.float32 and boxes.stride(1) == 1 and boxes.shape[1] >= ncols
    rois = torch.empty((n, ncols + 1), dtype=torch.float32, device='cuda')
    L.call('dt_scale_rois', C.c_void_p(boxes.data_ptr()), boxes.stride(0), n, ncols, L.ptr(batch_idx), int(per_image),
           float(im_scale), L.ptr(rois), L.stream_ptr())
    return rois


def pairs_to_f16(x):
    """bf16 pair rows [..., 2C] -> fp16 [..., C] = fp16(hi + lo): the operand of a DT_DTYPE_F16 conv."""
    torch = L.require_cuda()
    assert x.dtype == torch.bfloat16 and x.is_contiguous() and x.shape[-1] % 16 == 0
    Cc = x.shape[-1] // 2
    out = torch.empty(tuple(x.shape[:-1]) + (Cc,), dtype=torch.float16, device='cuda')
    L.call('dt_pairs_to_f16', L.ptr(x), x.numel() // x.shape[-1], Cc, L.ptr(out), L.stream_ptr())
    return out


def spatial_mean(x, round_tf32=False, x3=False):
    """x [N, H, W, C] -> [N, C]: mean over W, then over H (ReduceBackMean twice)."""
    torch = L.require_cuda()
    N, H, W, ld = x.shape
    Cc = ld // 2 if x3 else ld
    y = torch.empty((N, ld), dtype=x.dtype, device='cuda')
    L.call('dt_spatial_mean', L.ptr(x), N, H, W, Cc, ld, int(x.dtype == torch.float32), int(bool(round_tf32)), int(bool(x3)),
           L.ptr(y), ld, L.stream_ptr())
    return y


def time_mean(x, round_tf32=False, x3=False):
    """x [B, T, H, W, ld] -> [B, 1, H, W, ld]: mean over the frames (the 'avg' body/head link)."""
    torch = L.require_cuda()
    B, T, H, W, ld = x.shape
    assert x.is_contiguous()
    Cc = ld // 2 if x3 else ld
    y = torch.empty((B, 1, H, W, ld), dtype=x.dtype, device='cuda')
    L.call('dt_time_mean', L.ptr(x), B, T, H * W, Cc, ld, int(x.dtype == torch.float32), int(bool(round_tf32)), int(bool(x3)),
           L.ptr(y), ld, L.stream_ptr())
    return y


def fold_tube_heads(o, R, T, C):
    """o [R*T, ld] fp32 = per-frame [cls | bbox] -> (cls [R, C], bbox [R, C*T*4])."""
    torch = L.require_cuda()
    cls = torch.empty((R, C), dtype=torch.float32, device='cuda')
    bbox = torch.empty((R, C * T * 4), dtype=torch.float32, device='cuda')
    assert o.dtype == torch.float32 and o.stride(1) == 1
    L.call('dt_fold_tube_heads', L.ptr(o), o.stride(0), R, T, C, L.ptr(cls), L.ptr(bbox),
           L.stream_ptr())
    return cls, bbox


def aug_scale_rois(boxes, im_scale, flip=False, im_hw=None, per_image=1):
    """A test-time view's keypoint RoIs (lib/core/test.py:630-684): boxes [n, >=4] fp32 (row stride free) ->
    rois [n, 5] = (i // per_image, flip_boxes(boxes) * im_scale), the flip with the width im_hw[i // per_image, 1].
    Without the flip this is scale_rois(boxes, 4, im_scale, per_image=per_image)."""
    torch = L.require_cuda()
    n = boxes.shape[0]
    assert boxes.dtype == torch.float32 and boxes.stride(1) == 1 and boxes.shape[1] >= 4
    assert not flip or (im_hw is not None and im_hw.dtype == torch.float32 and im_hw.shape[1] == 2 and im_hw.is_contiguous())
    rois = torch.empty((n, 5), dtype=torch.float32, device='cuda')
    w = C.c_void_p(im_hw.data_ptr() + 4) if flip else None
    L.call('dt_aug_scale_rois', C.c_void_p(boxes.data_ptr()), boxes.stride(0), n, int(bool(flip)), w, 2, int(per_image),
           float(im_scale), L.ptr(rois), L.stream_ptr())
    return rois


def keypoint_decode_aug(lowres, flips, perm, hm_max, boxes, K=17, min_size=0, want_heatmaps=False):
    """keypoint_decode of V test-time views combined (lib/core/test.py:686-747), 2-D heads: lowres [V, D, S, S, >=4K]
    fp32, flips [V], perm [K] (flip_heatmaps' joint swap), hm_max (HM_MAX, else HM_AVG).
    Returns (xy_preds [D, 4, K], combined heatmaps [D, K, 4S, 4S] or None)."""
    torch = L.require_cuda()
    V, D, S, _, ldl = lowres.shape
    assert V == len(flips) and len(perm) == K
    assert lowres.dtype == torch.float32 and lowres.is_contiguous()
    assert boxes.stride(1) == 1 and boxes.dtype == torch.float32
    xy = L.zeros((D, 4, K), torch.float32)
    heat = L.zeros((D, K, 4 * S, 4 * S), torch.float32) if want_heatmaps else None
    L.call('dt_keypoint_decode_aug', L.ptr(lowres), D * S * S * ldl, ldl, S, K, V, (C.c_int * V)(*[int(bool(f)) for f in flips]),
           (C.c_int * K)(*[int(p) for p in perm]), int(bool(hm_max)), C.c_void_p(boxes.data_ptr()), boxes.stride(0), None, D,
           int(min_size), L.ptr(heat), L.ptr(xy), L.stream_ptr())
    return xy, heat
