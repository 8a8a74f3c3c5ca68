"""H100 execution engine for the reference's keypoint R-CNN graphs.

What the reference runs as three Caffe2 nets with host ops in between
(lib/core/test.py:158-252,584-627,897-958; SURVEY.md §3.1) runs here as one stream of
kernel launches with no host round trip between the image blob and the detections:

  prep_clip -> conv1 -> pool1 -> res2..res5 (wgmma implicit GEMM, fused affine/ReLU/residual)
  -> FPN (lateral 1x1 with the top-down upsample-add in the epilogue, post-hoc convs, P6)
  -> [body/head link: centre-frame slice]
  -> per level: RPN 3x3 + fused (cls|bbox) 1x1 -> device top-k/decode -> batched bitmask NMS
  -> collect / distribute -> RoIAlign (levels + un-shuffle fused) -> fc6/fc7/(cls|bbox) GEMMs
  -> softmax/decode/clip -> per-class NMS -> DETECTIONS_PER_IM limit
  -> keypoint RoIAlign -> 8 x conv3x3 -> sub-pixel deconv -> bilinear 2x + cubic decode

Layout: NDHWC ([B, T, H, W, C]); T is an outer stride, so the reference's
MoveTimeToBatch/Channel shuffles (lib/modeling/detector.py:467-557) cost nothing.
Supported graphs this round: FPN / FPN3D ResNet-{50,101,152} conv5 bodies with 2-D heads
(BODY_HEAD_LINK 'slice-center', or 2-D models), head_builder.add_roi_2mlp_head and
keypoint_rcnn_heads.add_roi_pose_head_v1convX — the reference's runnable FPN semantics
(lib/modeling/FPN3D.py:228 raises for 3-D FPN heads).
"""
import numpy as np

from .. import _lib as L
from ..ops import conv as cv
from ..ops import box_ops, rpn_ops, dense_ops
from . import params as P
from .generate_anchors import generate_anchors


class _Conv(object):
    """One packed convolution (+ fused epilogue parameters) resident on the device."""

    def __init__(self, torch, w, dtype, scale=None, bias=None, stride=(1, 1, 1), pad=(0, 0, 0), relu=False):
        w = torch.from_numpy(np.ascontiguousarray(w))
        if w.dim() == 2:
            k = (1, 1, 1)
        elif w.dim() == 4:
            k = (1, w.shape[2], w.shape[3])
        else:
            k = tuple(w.shape[2:])
        self.k, self.stride, self.pad, self.relu, self.dtype = k, stride, pad, relu, dtype
        self.w = cv.pack_weight(w, dtype)
        self.cout = w.shape[0]
        self.scale = torch.from_numpy(np.ascontiguousarray(scale, dtype=np.float32)).cuda() if scale is not None else None
        self.bias = torch.from_numpy(np.ascontiguousarray(bias, dtype=np.float32)).cuda() if bias is not None else None

    def __call__(self, x, residual=None, res_mode=0, relu=None, out_f32=None, cin=None, out=None, time_major=False,
                 out_frames=None):
        return cv.conv3d(x, self.w, self.k, self.stride, self.pad, self.scale, self.bias, residual, res_mode,
                         self.relu if relu is None else relu, out_f32=out_f32, dtype=self.dtype, cin=cin, out=out,
                         time_major=time_major, out_frames=out_frames)


class DetectionEngine(object):
    def __init__(self, cfg, blobs, spec=None, dtype='bf16'):
        torch = L.require_cuda()
        L.lib()
        self.torch = torch
        self.cfg = cfg
        self.spec = spec or P.GraphSpec(cfg)
        s = self.spec
        if s.fpn and s.head3d:
            raise NotImplementedError('3-D FPN heads are unimplemented in the reference too (FPN3D.py:228)')
        if not s.fpn and not s.head3d:
            raise NotImplementedError('engine: single-level bodies are wired for 3-D heads (BODY_HEAD_LINK \'\') only')
        if s.link not in ('slice-center', 'avg', 'none2d', ''):
            raise NotImplementedError('engine: BODY_HEAD_LINK %r' % s.link)
        # 'bf16x3': the parity mode (default of the drop-in surface): activations / weights as [hi | lo] bf16 pairs,
        # 3 bf16 MMAs per k-block -> 16 mantissa bits, <= 1e-3 end to end (tests) at the full kind::f16 MMA rate;
        # 'tf32x3': the same scheme on tf32 pairs (fp32 storage, ~21 bits, half MMA rate, twice the bytes);
        # 'tf32': fp32 storage, one tf32 MMA (1e-3 per layer, ~1.5e-3 end to end); 'bf16': fast, ~1e-2 end to end;
        # 'bf16x3h': bf16x3 everywhere except the four post-hoc FPN convs (the largest single kernels), which run as ONE
        # fp16 MMA per product on fp16 copies of the inner maps — 11-bit operands on one layer of any path
        self.dtype_name = dtype
        self.dtype = cv.MODE_NAMES[dtype]
        self.x3 = self.dtype in cv.SPLIT_MODES
        self.fp16_posthoc = dtype == 'bf16x3h'
        self.act_dtype = torch.bfloat16 if dtype.startswith('bf16') else torch.float32
        self.cin_pad = 8 if dtype.startswith('bf16') else 4
        self.skip_dead_frames = False       # compute only the consumed (centre) frame of the post-hoc FPN convs
        self._geom = {}
        self._build(blobs)

    # ------------------------------------------------------------------ weights
    def _c(self, blobs, name, affine=None, bias=False, **kw):
        scale = blobs[affine + '_s'] if affine else None
        b = blobs[affine + '_b'] if affine else (blobs[name + '_b'] if bias else None)
        return _Conv(self.torch, blobs[name + '_w'], self.dtype, scale, b, **kw)

    def _block(self, blobs, pre, dim_in, dim_out, st, tk):
        """One residual block (ResNet3D.py:21-152); the last conv carries the fused shortcut add + ReLU."""
        s = self.spec
        sc = self._c(blobs, pre + '_branch1', pre + '_branch1_bn', stride=st) if dim_in != dim_out else None
        if s.block == 'bottleneck':
            s1, s3 = (st, (1, 1, 1)) if s.stride_1x1 else ((1, 1, 1), st)
            return dict(sc=sc, convs=[
                self._c(blobs, pre + '_branch2a', pre + '_branch2a_bn', stride=s1, relu=True),
                self._c(blobs, pre + '_branch2b', pre + '_branch2b_bn', stride=s3, pad=(tk // 2, 1, 1), relu=True),
                self._c(blobs, pre + '_branch2c', pre + '_branch2c_bn', relu=True)])
        return dict(sc=sc, convs=[
            self._c(blobs, pre + '_branch2a', pre + '_branch2a_bn', stride=st, pad=(tk // 2, 1, 1), relu=True),
            self._c(blobs, pre + '_branch2b', pre + '_branch2b_bn', pad=(tk // 2, 1, 1), relu=True)])

    @staticmethod
    def _run_block(blk, y):
        sc = blk['sc'](y) if blk['sc'] is not None else y
        h = y
        for c in blk['convs'][:-1]:
            h = c(h)
        return blk['convs'][-1](h, residual=sc, res_mode=1)

    def _build(self, blobs):
        s, cfg, torch = self.spec, self.cfg, self.torch
        # conv1: 7x7/2 on the 3-channel blob with the filter row packed into K (dt_conv1_7x7s2)
        w1 = torch.from_numpy(np.ascontiguousarray(blobs['conv1_w']))
        # conv1: tf32x3 runs it as exact fp32 FMAs; bf16x3 on the tensor cores over a split-pixel blob
        self.conv1_exact = self.dtype == cv.TF32X3
        self.conv1_w = cv.pack_conv1_weight_f32(w1) if self.conv1_exact else cv.pack_conv1_weight(w1, self.dtype)
        self.conv1_s = torch.from_numpy(np.ascontiguousarray(blobs['res_conv1_bn_s'], dtype=np.float32)).cuda()
        self.conv1_b = torch.from_numpy(np.ascontiguousarray(blobs['res_conv1_bn_b'], dtype=np.float32)).cuda()
        self.stages = []
        dim_in = s.dims[0]
        for si, n in enumerate(s.counts):
            dim_out = s.dims[si + 1]
            tk = 1 if si == 0 else s.tk_body
            blocks = []
            for i in range(n):
                pre = 'res%d_%d' % (si + 2, i)
                stride = 2 if (dim_in != dim_out and si != 0) else 1
                st = (1, stride, stride)
                blocks.append(self._block(blobs, pre, dim_in, dim_out, st, tk))
                dim_in = dim_out
            self.stages.append(blocks)
        self.pixel_means = np.asarray(cfg.PIXEL_MEANS, dtype=np.float32).ravel()
        if s.fpn:
            self._build_fpn_heads(blobs)
        else:
            self._build_tube_heads(blobs, dim_in)
        self._build_keypoint_head(blobs)

    def _build_fpn_heads(self, blobs):
        s, cfg, torch = self.spec, self.cfg, self.torch
        names = s.stage_blobs[::-1]
        self.fpn_inner = [self._c(blobs, 'fpn_inner_' + names[0], bias=True)]
        for i in range(1, len(names)):
            self.fpn_inner.append(self._c(blobs, 'fpn_inner_%s_lateral' % names[i], bias=True))
        tk = s.tk_body
        self.fpn_out = [self._c(blobs, 'fpn_' + n, bias=True, pad=(tk // 2, 1, 1)) for n in names]
        if self.fp16_posthoc:
            self.fpn_out = [_Conv(torch, blobs['fpn_%s_w' % n], cv.F16, None, blobs['fpn_%s_b' % n], pad=(tk // 2, 1, 1)) for n in names]
        # RPN (shared across levels): 3x3 + fused [cls | bbox] 1x1
        k = str(s.rpn_levels[0])
        A = s.num_anchors
        self.rpn_conv = self._c(blobs, 'conv_rpn_fpn' + k, bias=True, pad=(0, 1, 1), relu=True)
        w = np.concatenate([blobs['rpn_cls_logits_fpn%s_w' % k], blobs['rpn_bbox_pred_fpn%s_w' % k]], 0)
        b = np.concatenate([blobs['rpn_cls_logits_fpn%s_b' % k], blobs['rpn_bbox_pred_fpn%s_b' % k]], 0)
        self.rpn_out = _Conv(torch, w, self.dtype, None, b)
        self.rpn_out_ld = (5 * A + 3) // 4 * 4
        self.anchors = [torch.from_numpy(generate_anchors(
            stride=2. ** lvl, sizes=(cfg.FPN.RPN_ANCHOR_START_SIZE * 2. ** (lvl - s.rpn_levels[0]),),
            aspect_ratios=cfg.FPN.RPN_ASPECT_RATIOS, time_dim=1)).cuda() for lvl in s.rpn_levels]
        # box head: fc6 columns permuted from (c, h, w) to the RoIAlign output order (h, w, c)
        res = cfg.FAST_RCNN.ROI_XFORM_RESOLUTION
        fd = s.fpn_dim
        w6 = blobs['fc6_w'].reshape(-1, fd, res, res).transpose(0, 2, 3, 1).reshape(blobs['fc6_w'].shape[0], -1)
        self.fc6 = _Conv(torch, w6, self.dtype, None, blobs['fc6_b'], relu=True)
        self.fc7 = self._c(blobs, 'fc7', bias=True, relu=True)
        wcb = np.concatenate([blobs['cls_score_w'], blobs['bbox_pred_w']], 0)
        bcb = np.concatenate([blobs['cls_score_b'], blobs['bbox_pred_b']], 0)
        self.cls_bbox = _Conv(torch, wcb, self.dtype, None, bcb)
        self.cls_bbox_ld = (5 * s.num_classes + 3) // 4 * 4

    def _build_tube_heads(self, blobs, dim_conv):
        """Single-level 3-D RPN (model_builder.py:500-609) and the res5 RoI head + 3-D outputs
        (ResNet3D.py:301-327, model_builder.py:427-473)."""
        s, cfg, torch = self.spec, self.cfg, self.torch
        T = s.T_head
        tk = cfg.VIDEO.TIME_KERNEL_DIM.HEAD_RPN
        A = s.num_anchors
        self.feat_stride = 16.0
        self.rpn_conv = self._c(blobs, 'conv_rpn', bias=True, pad=(tk // 2, 1, 1), relu=True)
        w = np.concatenate([blobs['rpn_cls_logits_1_w'], blobs['rpn_bbox_pred_1_w']], 0)
        b = np.concatenate([blobs['rpn_cls_logits_1_b'], blobs['rpn_bbox_pred_1_b']], 0)
        self.rpn_out = _Conv(torch, w, self.dtype, None, b)
        self.rpn_out_ld = (5 * A + 3) // 4 * 4
        self.anchors = [torch.from_numpy(generate_anchors(stride=self.feat_stride, sizes=cfg.RPN.SIZES,
                                                          aspect_ratios=cfg.RPN.ASPECT_RATIOS, time_dim=T)).cuda()]
        arch = s.roi_head.split('add_')[1].split('_')[0]
        n5, dout = P._BLOCKS[arch][0][3], P._BLOCKS[arch][2][4]
        stride_init = int(cfg.FAST_RCNN.ROI_XFORM_RESOLUTION / 7)
        self.res5 = []
        din = dim_conv
        for i in range(n5):
            st = stride_init if din != dout else 1              # add_bottleneck_block: stage_id 4, dim change
            self.res5.append(self._block(blobs, 'res5_%d' % i, din, dout, (1, st, st), 1))
            din = dout
        wcb = np.concatenate([blobs['cls_score_1_w'], blobs['bbox_pred_1_w']], 0).reshape(-1, dout)
        bcb = np.concatenate([blobs['cls_score_1_b'], blobs['bbox_pred_1_b']], 0)
        self.cls_bbox = _Conv(torch, wcb, self.dtype, None, bcb)
        self.cls_bbox_ld = (5 * s.num_classes + 3) // 4 * 4

    def _build_keypoint_head(self, blobs):
        s, cfg, torch = self.spec, self.cfg, self.torch
        self.kps_convs = []
        if cfg.MODEL.KEYPOINTS_ON:
            tkk = cfg.VIDEO.TIME_KERNEL_DIM.HEAD_KPS if s.kps_head.endswith('_3d') else 1
            for i in range(cfg.KRCNN.NUM_STACKED_CONVS):
                ks = cfg.KRCNN.CONV_HEAD_KERNEL
                self.kps_convs.append(self._c(blobs, 'conv_fcn%d' % (i + 1), bias=True, pad=(tkk // 2, ks // 2, ks // 2), relu=True))
            wt = blobs['kps_score_lowres_w']                 # ConvTranspose (Cin, K, 4, 4), stride 2, pad 1
            cin, K = wt.shape[0], wt.shape[1]
            w3 = np.zeros((4 * K, cin, 3, 3), np.float32)     # four 2x2 sub-pixel filters on a 3x3 footprint
            for py in range(2):
                for px in range(2):
                    for dy in (-1, 0, 1):
                        ky = py + 1 - 2 * dy
                        if not 0 <= ky <= 3:
                            continue
                        for dx in (-1, 0, 1):
                            kx = px + 1 - 2 * dx
                            if not 0 <= kx <= 3:
                                continue
                            w3[(py * 2 + px) * K:(py * 2 + px + 1) * K, :, dy + 1, dx + 1] = wt[:, :, ky, kx].T
            self.kps_lowres = _Conv(torch, w3, self.dtype, None, np.tile(blobs['kps_score_lowres_b'], 4), pad=(0, 1, 1))

    # ------------------------------------------------------------------ backbone
    def body(self, x):
        """x [B,T,2,(Hp+6)/2,Wp+8,cin_pad] (zero-bordered blob, rows split by parity) -> stage outputs (finest first)."""
        torch = self.torch
        B, T = x.shape[:2]
        if self.conv1_exact:      # exact fp32 conv1 on the raw (un-bordered) blob
            y = cv.conv1_7x7s2_f32(x.view((B * T,) + tuple(x.shape[2:])), self.conv1_w, self.conv1_s, self.conv1_b)
        else:
            hp, wp = 2 * x.shape[3] - 6, x.shape[4] - 8
            y = cv.conv1_7x7s2(x.view((B * T,) + tuple(x.shape[2:])), self.conv1_w, (hp, wp), self.conv1_s, self.conv1_b,
                               relu=True, dtype=self.dtype)
        y = dense_ops.maxpool2d(y, 3, 2, 1, x3=self.x3)
        y = y.view((B, T) + tuple(y.shape[1:]))
        outs = []
        for blocks in self.stages:
            for blk in blocks:
                y = self._run_block(blk, y)
            outs.append(y)
        return outs

    def fpn(self, stage_outs):
        """-> FPN maps finest first: [P2, P3, P4, P5, P6], each [B, Tout, h, w, 256]."""
        s = self.spec
        coarse_first = stage_outs[::-1]
        inner = [self.fpn_inner[0](coarse_first[0])]
        for i in range(1, len(coarse_first)):
            inner.append(self.fpn_inner[i](coarse_first[i], residual=inner[i - 1], res_mode=2))
        outs = []
        for i, x in enumerate(inner):
            tm = s.link == 'slice-center' and x.shape[1] > 1
            if self.fp16_posthoc:
                x16 = dense_ops.pairs_to_f16(x)
                c = int(self.cfg.VIDEO.NUM_FRAMES_MID / 2)
                of = (c, 1) if (self.skip_dead_frames and tm) else None
                outs.append(cv.conv3d(x16, self.fpn_out[i].w, self.fpn_out[i].k, (1, 1, 1), self.fpn_out[i].pad, None, self.fpn_out[i].bias,
                                      dtype=cv.F16, split_out=True, time_major=(tm and of is None), out_frames=of))
                continue
            if self.skip_dead_frames and s.link == 'slice-center' and x.shape[1] > 1:
                # only the frame the link slices is consumed: compute just that output frame
                c = int(self.cfg.VIDEO.NUM_FRAMES_MID / 2)
                y = self.fpn_out[i](x, out_frames=(c, 1))
            else:
                # frames-outermost output: the centre-frame link below is then a view, not a gather
                y = self.fpn_out[i](x, time_major=(s.link == 'slice-center' and x.shape[1] > 1))
            outs.append(y)
        p5 = outs[0]
        B, T = p5.shape[:2]
        if p5.is_contiguous():
            p6 = dense_ops.maxpool2d(p5.view((B * T,) + tuple(p5.shape[2:])), 1, 2, 0, x3=self.x3)
            outs.insert(0, p6.view((B, T) + tuple(p6.shape[1:])))
        else:                               # frames-outermost storage: pool the [T, B] stack, present [B, T]
            p5t = p5.permute(1, 0, 2, 3, 4)
            assert p5t.is_contiguous()
            p6 = dense_ops.maxpool2d(p5t.view((T * B,) + tuple(p5.shape[2:])), 1, 2, 0, x3=self.x3)
            outs.insert(0, p6.view((T, B) + tuple(p6.shape[1:])).permute(1, 0, 2, 3, 4))
        return outs[::-1]

    def link(self, feats):
        """model_builder.time_pool_blobs (:1024-1042): centre-frame slice or mean over T -> [B, 1, h, w, C]."""
        s = self.spec
        if s.head3d:
            return feats
        out = []
        for f in feats:
            if f.shape[1] == 1:
                out.append(f)
                continue
            if s.link == 'avg':             # TimePool 'avg': mean over the frames
                out.append(dense_ops.time_mean(f, round_tf32=(self.dtype == cv.TF32), x3=self.x3))
                continue
            c = int(self.cfg.VIDEO.NUM_FRAMES_MID / 2)
            v = f[:, c:c + 1]
            out.append(v if v.is_contiguous() else v.contiguous())
        return out

    # ------------------------------------------------------------------ heads
    def rpn(self, feats2d, im_info):
        """feats2d finest first [P2..P6] as [B,1,h,w,C].  Returns rois [B,R,5], roi_counts [B]."""
        torch, cfg, s = self.torch, self.cfg, self.spec
        B = feats2d[0].shape[0]
        Lv = len(feats2d)
        K = cfg.TEST.RPN_PRE_NMS_TOP_N
        A = s.num_anchors
        props = L.zeros((B, Lv, K, 5), torch.float32)
        counts = L.zeros((B, Lv), torch.int32)
        levels = []
        for l, f in enumerate(feats2d):
            h = self.rpn_conv(f)
            Bq, _, H, W, _ = h.shape
            o = torch.empty((Bq, 1, H, W, self.rpn_out_ld), dtype=torch.float32, device='cuda')
            self.rpn_out(h, out_f32=True, out=o)
            o4 = o.view(Bq, H, W, self.rpn_out_ld)
            levels.append(dict(logits=o4[..., :A], deltas=o4[..., A:5 * A], anchors=self.anchors[l],
                               feat_stride=2. ** s.rpn_levels[l], out=props[:, l], counts=counts[:, l]))
        rpn_ops.rpn_proposals_levels(levels, im_info, K, A, float(cfg.TEST.RPN_MIN_SIZE), 1)      # all levels, one launch
        keep, nkeep = box_ops.nms_batched(props.view(B * Lv, K, 5), counts.view(-1), cfg.TEST.RPN_NMS_THRESH,
                                          box_ops.NMS_2D_GE, box_ops.ORDER_INDEX, max_keep=cfg.TEST.RPN_POST_NMS_TOP_N)
        return rpn_ops.collect(props, keep, nkeep, cfg.TEST.RPN_POST_NMS_TOP_N)

    def _roi_feats(self, feats2d, rois_flat, resolution, sampling, planar=False):
        s = self.spec
        nl = len(s.roi_levels)
        fl = [f.view((f.shape[0] * f.shape[1],) + tuple(f.shape[2:])) for f in feats2d[:nl]]
        scales = [1. / 2 ** lvl for lvl in s.roi_levels]
        levels, _, _ = rpn_ops.distribute(rois_flat, None, col0=1, T=1, k_min=s.roi_levels[0], k_max=s.roi_levels[-1],
                                          s0=float(self.cfg.FPN.ROI_CANONICAL_SCALE), lvl0=float(self.cfg.FPN.ROI_CANONICAL_LEVEL),
                                          want_restore=False)
        return dense_ops.roi_align(fl, scales, rois_flat, levels, resolution, sampling, T=1, k_min=s.roi_levels[0],
                                   round_tf32=(self.dtype == cv.TF32), x3_mode=(2 if planar else 1) if self.x3 else 0)

    def box_head(self, feats2d, rois, roi_counts, im_info, im_hw):
        torch, cfg, s = self.torch, self.cfg, self.spec
        B, R, _ = rois.shape
        C = s.num_classes
        x = self._roi_feats(feats2d, rois.view(B * R, 5), cfg.FAST_RCNN.ROI_XFORM_RESOLUTION,
                            cfg.FAST_RCNN.ROI_XFORM_SAMPLING_RATIO, planar=True)      # x3: [hi block | lo block] rows for the FC
        x = x.view(1, 1, 1, B * R, -1)
        x = self.fc7(self.fc6(x))
        o = torch.empty((1, 1, 1, B * R, self.cls_bbox_ld), dtype=torch.float32, device='cuda')
        self.cls_bbox(x, out_f32=True, out=o)
        o2 = o.view(B * R, self.cls_bbox_ld)
        dets, cnt = rpn_ops.box_decode(rois, roi_counts, o2[:, :C], o2[:, C:5 * C], C, im_info, im_hw,
                                       cfg.MODEL.BBOX_REG_WEIGHTS, cfg.TEST.SCORE_THRESH, 1)
        keep, nkeep = box_ops.nms_batched(dets.view(B * (C - 1), R, 5), cnt, cfg.TEST.NMS, box_ops.NMS_2D_GE,
                                          box_ops.ORDER_INDEX)
        return rpn_ops.limit_detections(dets, keep, nkeep, cfg.TEST.DETECTIONS_PER_IM, cap=min(R, self.det_cap))

    def keypoint_head(self, feats, boxes, batch_idx, im_scale, want_heatmaps=False, per_image=1):
        """boxes [D, >= 4*Th] image space (fp32 cuda, any row stride), batch_idx [D] fp32 (or None: image index =
        row // per_image) -> xy_preds [D, 4, Th*K].
        2-D heads: feats = per-level centre-frame maps; tube heads: feats = [conv feature 5-D]."""
        torch, cfg, s = self.torch, self.cfg, self.spec
        D = boxes.shape[0]
        Th = s.T_head
        # _get_rois_blob (test.py:76-113): float64 product, stored fp32, image index in col 0
        rois = dense_ops.scale_rois(boxes, 4 * Th, im_scale, batch_idx, per_image)
        res, samp = cfg.KRCNN.ROI_XFORM_RESOLUTION, cfg.KRCNN.ROI_XFORM_SAMPLING_RATIO
        if s.head3d:
            x = self._roi_feats_tube(feats[0], rois, res, samp)               # [D, Th, S, S, C]
        else:
            x = self._roi_feats(feats, rois, res, samp)
            x = x.view((D, 1) + tuple(x.shape[2:]))
        for c in self.kps_convs:
            x = c(x)
        S = x.shape[2]
        ld = (4 * s.K + 3) // 4 * 4
        low = torch.empty((D, Th, S, S, ld), dtype=torch.float32, device='cuda')
        self.kps_lowres(x, out_f32=True, out=low)                             # per-frame (kT = 1): time in batch
        return dense_ops.keypoint_decode(low.view(D * Th, S, S, ld), boxes, s.K, Th,
                                         min_size=cfg.KRCNN.INFERENCE_MIN_SIZE, want_heatmaps=want_heatmaps)

    # ------------------------------------------------------------------ tube (3-D) heads
    def _roi_feats_tube(self, feat5d, rois, resolution, sampling):
        """RoIFeatureTransform for 3-D heads (detector.py:216-254): tube -> per-frame boxes with image
        index b*T + t, 2-D RoIAlign, back to [R, T, P, P, C]."""
        B, T = feat5d.shape[:2]
        f = feat5d.view((B * T,) + tuple(feat5d.shape[2:]))
        return dense_ops.roi_align([f], [1.0 / self.feat_stride], rois, None, resolution, sampling, T=T,
                                   round_tf32=(self.dtype == cv.TF32), x3_mode=1 if self.x3 else 0)

    def rpn_tube(self, feat5d, im_info):
        """Single-level 3-D RPN -> rois [B, R, 4T+1], roi_counts [B]."""
        torch, cfg, s = self.torch, self.cfg, self.spec
        B, T, H, W, _ = feat5d.shape
        A, K = s.num_anchors, cfg.TEST.RPN_PRE_NMS_TOP_N
        h = self.rpn_conv(feat5d)
        o = torch.empty((B, T, H, W, self.rpn_out_ld), dtype=torch.float32, device='cuda')
        self.rpn_out(h, out_f32=True, out=o)
        n = H * W * A
        Kc = n if (K <= 0 or K > n) else K
        props = L.zeros((B, 1, Kc, 4 * T + 1), torch.float32)
        counts = L.zeros((B, 1), torch.int32)
        rpn_ops.rpn_proposals(o[..., :A], o[..., A:5 * A], self.anchors[0], self.feat_stride, im_info, K,
                              float(cfg.TEST.RPN_MIN_SIZE), T, out=props[:, 0], counts=counts[:, 0], time_major=True)
        keep, nkeep = box_ops.nms_batched(props.view(B, Kc, 4 * T + 1), counts.view(-1), cfg.TEST.RPN_NMS_THRESH,
                                          box_ops.NMS_TUBE_GT if T > 1 else box_ops.NMS_2D_GE,
                                          box_ops.ORDER_SCORE if T > 1 else box_ops.ORDER_INDEX,
                                          max_keep=cfg.TEST.RPN_POST_NMS_TOP_N)
        return rpn_ops.collect(props, keep, nkeep, cfg.TEST.RPN_POST_NMS_TOP_N)

    def box_head_tube(self, feat5d, rois, roi_counts, im_info, im_hw):
        torch, cfg, s = self.torch, self.cfg, self.spec
        B, R, ldr = rois.shape
        T, C = s.T_head, s.num_classes
        x = self._roi_feats_tube(feat5d, rois.view(B * R, ldr), cfg.FAST_RCNN.ROI_XFORM_RESOLUTION,
                                 cfg.FAST_RCNN.ROI_XFORM_SAMPLING_RATIO)                 # [BR, T, 7, 7, C]
        for blk in self.res5:
            x = self._run_block(blk, x)
        n, _, hh, ww, ch = x.shape
        x = dense_ops.spatial_mean(x.view(n * T, hh, ww, ch), round_tf32=(self.dtype == cv.TF32), x3=self.x3)    # [BR*T, C]
        o = torch.empty((1, 1, 1, n * T, self.cls_bbox_ld), dtype=torch.float32, device='cuda')
        self.cls_bbox(x.view(1, 1, 1, n * T, ch), out_f32=True, out=o)
        cls, bbox = dense_ops.fold_tube_heads(o.view(n * T, self.cls_bbox_ld), n, T, C)
        dets, cnt = rpn_ops.box_decode(rois, roi_counts, cls, bbox, C, im_info, im_hw, cfg.MODEL.BBOX_REG_WEIGHTS,
                                       cfg.TEST.SCORE_THRESH, T)
        keep, nkeep = box_ops.nms_batched(dets.view(B * (C - 1), R, 4 * T + 1), cnt, cfg.TEST.NMS,
                                          box_ops.NMS_TUBE_GT if T > 1 else box_ops.NMS_2D_GE,
                                          box_ops.ORDER_SCORE if T > 1 else box_ops.ORDER_INDEX)
        return rpn_ops.limit_detections(dets, keep, nkeep, cfg.TEST.DETECTIONS_PER_IM, cap=min(R, self.det_cap))

    # ------------------------------------------------------------------ end to end
    def blob_geometry(self, h, w):
        """prep_im_for_blob / im_list_to_blob geometry (blob.py:40-90): scale, resized, padded size."""
        cfg = self.cfg
        target = cfg.TEST.SCALES[0]
        smin, smax = min(h, w), max(h, w)
        scale = float(target) / float(smin)
        if np.round(scale * smax) > cfg.TEST.MAX_SIZE:
            scale = float(cfg.TEST.MAX_SIZE) / float(smax)
        if scale == 1.0:
            hr, wr = h, w
        else:
            hr, wr = int(round(h * scale)), int(round(w * scale))     # cv2: saturate_cast<int>(size * fx)
        stride = float(cfg.FPN.COARSEST_STRIDE) if cfg.FPN.FPN_ON else 1.0
        hp, wp = int(np.ceil(hr / stride) * stride), int(np.ceil(wr / stride) * stride)
        return scale, (hr, wr), (hp, wp)

    def plain(self, t):
        """Activation tensor as plain values (joins the [hi | lo] pairs of the 3xTF32 mode)."""
        return cv.join_split(t) if self.x3 else t

    def _blob(self, frames_u8, scale, hr, wr, hp, wp):
        """uint8 frames -> network input: zero-bordered bf16 / tf32 blob for the packed-row conv1, or the raw
        fp32 blob for the exact conv1 of the 3xTF32 mode."""
        B, T, H, W, _ = frames_u8.shape
        # conv1 (7x7 / 2, pad 3) yields ceil(h / 2) rows; the kernels want an even physical blob, so an odd blob size
        # (single-level bodies do no /32 padding: a 1280x720 frame gives 750x1333) gets one more zero row / column.
        # That equals the conv's own zero padding, and im_info keeps the reference's (unpadded) blob size.
        hp, wp = hp + (hp & 1), wp + (wp & 1)
        if self.conv1_exact:
            x = dense_ops.prep_clip(frames_u8.view(B * T, H, W, 3), self.pixel_means, scale, (hr, wr), (hp, wp),
                                    cpad=4, out_f32=2)
            return x.view(B, T, hp, wp, 4)
        mode = 3 if self.dtype == cv.BF16X3 else int(self.dtype == cv.TF32)
        x = dense_ops.prep_clip(frames_u8.view(B * T, H, W, 3), self.pixel_means, scale, (hr, wr), (hp, wp),
                                cpad=self.cin_pad, out_f32=mode, border=(3, 4), row_planes=True)
        return x.view(B, T, 2, (hp + 6) // 2, wp + 8, self.cin_pad)

    def forward_features(self, frames_u8):
        """frames [B, T, H, W, 3] uint8 cuda -> (feats2d finest first, im_info [B,3], scale)."""
        torch = self.torch
        B, T, H, W, _ = frames_u8.shape
        scale, (hr, wr), (hp, wp) = self.blob_geometry(H, W)
        x = self._blob(frames_u8, scale, hr, wr, hp, wp)
        feats = self.link(self.fpn(self.body(x))) if self.spec.fpn else [self.body(x)[-1]]
        im_info = torch.tensor([[hp, wp, scale]] * B, dtype=torch.float32, device='cuda')
        return feats, im_info, scale

    def _geom_tensors(self, B, H, W):
        """im_info / im_hw / batch indices for a (B, H, W) batch, created once (no H2D in the hot loop)."""
        key = (B, H, W)
        g = self._geom.get(key)
        if g is None:
            torch = self.torch
            scale, (hr, wr), (hp, wp) = self.blob_geometry(H, W)
            g = dict(scale=scale, hr=hr, wr=wr, hp=hp, wp=wp,
                     im_info=torch.tensor([[hp, wp, scale]] * B, dtype=torch.float32, device='cuda'),
                     im_hw=torch.tensor([[H, W]] * B, dtype=torch.float32, device='cuda'))
            self._geom[key] = g
        return g

    @property
    def det_cap(self):
        """Detection slots per clip: DETECTIONS_PER_IM (+ a few for exact score ties at the threshold,
        lib/core/test.py:796-800 keeps all of them)."""
        d = self.cfg.TEST.DETECTIONS_PER_IM
        return (d + 4 + 7) // 8 * 8 if d > 0 else self.cfg.TEST.RPN_POST_NMS_TOP_N

    def detect_static(self, frames_u8, want_heatmaps=False):
        """The whole path with NO host synchronisation (CUDA-graph capturable): fixed-capacity outputs
        plus device-side counts.  dets [B, C-1, cap, 5], det_counts [B*(C-1)], xy [B*cap, 4, K]."""
        torch, s = self.torch, self.spec
        B, T, H, W, _ = frames_u8.shape
        g = self._geom_tensors(B, H, W)
        x = self._blob(frames_u8, g['scale'], g['hr'], g['wr'], g['hp'], g['wp'])
        if s.fpn:
            feats = self.link(self.fpn(self.body(x)))
            rois, _, roi_counts = self.rpn(feats, g['im_info'])
            dets, det_counts = self.box_head(feats, rois, roi_counts, g['im_info'], g['im_hw'])
        else:
            feats = [self.body(x)[-1]]
            rois, _, roi_counts = self.rpn_tube(feats[0], g['im_info'])
            dets, det_counts = self.box_head_tube(feats[0], rois, roi_counts, g['im_info'], g['im_hw'])
        out = dict(dets=dets, det_counts=det_counts, xy=None, heat=None)
        if self.kps_convs:
            cap = dets.shape[2]
            if dets.shape[1] == 1:          # one foreground class: the detections ARE the keypoint boxes (a view)
                boxes = dets.view(B * cap, dets.shape[3])
            else:
                boxes = dets[:, 0].reshape(B * cap, dets.shape[3])
            out['xy'], out['heat'] = self.keypoint_head(feats, boxes, None, g['scale'], want_heatmaps, per_image=cap)
        return out

    def gather(self, out):
        """Host side of detect_static: per clip (boxes [n,5], keyps [n,4,K]) as device tensor views."""
        s = self.spec
        dets = out['dets']
        B, _, cap, _ = dets.shape
        cnt = out['det_counts'].view(B, s.num_classes - 1)[:, 0].tolist()
        if max(cnt) > cap:
            raise RuntimeError('more than %d detections tie at the DETECTIONS_PER_IM threshold (%s)' % (cap, cnt))
        res = []
        for b in range(B):
            n = cnt[b]
            res.append(dict(boxes=dets[b, 0, :n],
                            keyps=(out['xy'][b * cap:b * cap + n] if out['xy'] is not None else None),
                            heatmaps=(out['heat'][b * cap:b * cap + n] if out['heat'] is not None else None)))
        return res

    def detect(self, frames_u8, want_heatmaps=False):
        """Per clip dict(boxes [n,5], keyps [n,4,K], heatmaps) — the public per-batch call."""
        return self.gather(self.detect_static(frames_u8, want_heatmaps))

    # ------------------------------------------------------------------ CUDA graph
    def capture(self, B, T, H, W):
        """Capture detect_static for a fixed batch geometry.  Returns (static_input, run) where run()
        replays the graph and returns the static output dict."""
        torch = self.torch
        static_in = torch.zeros((B, T, H, W, 3), dtype=torch.uint8, device='cuda')
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):                                     # warm-up: lazy attribute / workspace setup
                self.detect_static(static_in)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            static_out = self.detect_static(static_in)

        def run():
            graph.replay()
            return static_out
        return static_in, run
