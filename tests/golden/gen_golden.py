"""Generate tests/golden/*.npz by running the REFERENCE's own python on seeded
inputs.  Runs only in the build container (needs /root/reference and
oracle/_ref built by oracle/build_ref.py); the .npz files are committed so the
GPU box never needs the reference.

    python tests/golden/gen_golden.py

What runs, unmodified, from /root/reference/lib (py2-only syntax never executes
on these paths):
    utils/cython_bbox.pyx, utils/cython_nms.pyx   (compiled: oracle/_ref)
    utils/boxes.py            bbox_overlaps, bbox_transform, clip_tiled_boxes
    nms/py_cpu_nms_tubes.py   py_cpu_nms_tubes
    core/nms_wrapper.py       nms
    modeling/generate_anchors.py
    modeling/FPN.py           map_rois_to_fpn_levels   (source-extracted: the module imports caffe2)
    ops/generate_proposals.py GenerateProposalsOp
    ops/collect_and_distribute_fpn_rpn_proposals.py   collect / distribute
    ops/roi_blob_transforms.py RoIToBatchFormatOp
Shims, all recorded here: ``np.float``/``np.int`` aliases (removed in numpy 2);
py2 ``b''`` option strings are decoded to str; ``cfg.BBOX_XFORM_CLIP`` is re-set to a python float so numpy-2 promotion keeps
the fp32 arithmetic numpy 1.14 (the reference's pin) used; caffe2 / pycocotools
imports are stubbed with empty modules (never called).
scipy.optimize.linear_sum_assignment goldens come from the installed scipy
(1.18.1), the reference's call at core/tracking_engine.py:237.
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = '/root/reference/lib'


def _setup_reference_imports():
    sys.path.insert(0, ROOT)
    sys.path.insert(0, REF)
    np.float = float
    np.int = int
    from oracle import build_ref
    assert build_ref.build(), 'reference not present'
    from oracle._ref import cython_bbox, cython_nms
    import utils  # reference package
    sys.modules['utils.cython_bbox'] = cython_bbox
    sys.modules['utils.cython_nms'] = cython_nms
    utils.cython_bbox = cython_bbox
    utils.cython_nms = cython_nms
    for name in ['caffe2', 'caffe2.python', 'pycocotools', 'pycocotools.mask', 'pycocotools.coco']:
        sys.modules.setdefault(name, types.ModuleType(name))
    from core.config import cfg
    cfg.BBOX_XFORM_CLIP = float(cfg.BBOX_XFORM_CLIP)

    def _decode(d):     # py2 b'..' == '..'; py3 needs str
        for k, v in d.items():
            if isinstance(v, dict):
                _decode(v)
            elif isinstance(v, bytes):
                d[k] = v.decode()
    _decode(cfg)
    return cfg


class Blob(object):
    """The tensor interface Caffe2 hands to python ops (.data/.shape/.reshape)."""

    def __init__(self, data=None):
        self.data = data

    @property
    def shape(self):
        return self.data.shape

    def reshape(self, shape):
        self.data = np.zeros(shape, dtype=np.float32)


def rand_boxes(rng, n, w=1333, h=800, smin=8, smax=400):
    x1 = rng.uniform(0, w - smin, n); y1 = rng.uniform(0, h - smin, n)
    bw = rng.uniform(smin, smax, n); bh = rng.uniform(smin, smax, n)
    return np.stack([x1, y1, np.minimum(x1 + bw, w - 1), np.minimum(y1 + bh, h - 1)], 1).astype(np.float32)


def rand_tubes(rng, n, T, **kw):
    b = rand_boxes(rng, n, **kw)
    parts = [b]
    for t in range(1, T):
        shift = rng.normal(0, 6, (n, 2))            # translate the box, keep it valid
        grow = np.abs(rng.normal(0, 2, (n, 2)))
        parts.append((parts[-1] + np.hstack([shift, shift + grow])).astype(np.float32))
    return np.hstack(parts).astype(np.float32)


def clustered(rng, n, T):
    """boxes in clusters so that NMS actually suppresses"""
    centers = rand_tubes(rng, max(n // 8, 1), T)
    idx = rng.integers(0, centers.shape[0], n)
    return (centers[idx] + rng.normal(0, 10, (n, 4 * T))).astype(np.float32)


def main():
    cfg = _setup_reference_imports()
    import utils.boxes as rbox
    from nms.py_cpu_nms_tubes import py_cpu_nms_tubes
    from core.nms_wrapper import nms as ref_nms
    from modeling.generate_anchors import generate_anchors
    rng = np.random.default_rng(20260922)
    out = {}

    # ---- IoU (2-D and tubes) -------------------------------------------------
    a, b = rand_boxes(rng, 257), rand_boxes(rng, 130)
    out['iou2d_a'], out['iou2d_b'] = a, b
    out['iou2d_out'] = rbox.bbox_overlaps(a, b)
    ta, tb = rand_tubes(rng, 97, 3), rand_tubes(rng, 64, 3)
    out['iou3_a'], out['iou3_b'] = ta, tb
    out['iou3_out'] = rbox.bbox_overlaps(ta, tb).astype(np.float32)
    # 5-column (score-carrying) boxes as the tracker passes them
    a5 = np.hstack([a[:50], rng.random((50, 1)).astype(np.float32)])
    b5 = np.hstack([b[:40], rng.random((40, 1)).astype(np.float32)])
    out['iou5_a'], out['iou5_b'] = a5, b5
    out['iou5_out'] = rbox.bbox_overlaps(a5, b5).astype(np.float32)

    # ---- NMS -----------------------------------------------------------------
    for name, n, T in [('nms2d', 1000, 1), ('nms2d_small', 37, 1), ('nmst3', 600, 3), ('nmst2', 129, 2)]:
        d = np.hstack([clustered(rng, n, T), rng.permutation(n)[:, None].astype(np.float32) / n + 0.0005])
        d = d.astype(np.float32)
        out[name + '_dets'] = d
        for th in (0.3, 0.5, 0.7):
            keep = ref_nms(d, th)
            out['%s_keep_%d' % (name, int(th * 10))] = np.asarray(keep, dtype=np.int64)
    d = out['nmst3_dets']
    assert list(out['nmst3_keep_5']) == list(py_cpu_nms_tubes(d, 0.5))

    # ---- anchors ---------------------------------------------------------------
    out['anchors_s16'] = generate_anchors(stride=16, sizes=(128, 256, 512), aspect_ratios=(0.5, 1, 2))
    out['anchors_default'] = generate_anchors()
    out['anchors_rpn12_T3'] = generate_anchors(stride=16, sizes=(64, 128, 256, 512), aspect_ratios=(0.5, 1, 2), time_dim=3)
    for lvl in range(2, 7):
        out['anchors_fpn%d' % lvl] = generate_anchors(
            stride=2. ** lvl, sizes=(32 * 2. ** (lvl - 2),), aspect_ratios=(0.5, 1, 2), time_dim=1)

    # ---- bbox_transform / clip -------------------------------------------------
    boxes = rand_boxes(rng, 300)
    deltas = (rng.normal(0, 0.5, (300, 8))).astype(np.float32)
    deltas[::17, 2] = 9.0   # exercises the BBOX_XFORM_CLIP branch
    out['xform_boxes'], out['xform_deltas'] = boxes, deltas
    out['xform_out_w10'] = rbox.bbox_transform(boxes, deltas, (10., 10., 5., 5.))
    pred = rbox.bbox_transform(boxes, deltas, (1., 1., 1., 1.))
    out['xform_out_w1'] = pred.copy()
    out['xform_clip'] = rbox.clip_tiled_boxes(pred.copy(), np.array([800, 1333], dtype=np.float32))
    tboxes = rand_tubes(rng, 200, 3)
    tdeltas = rng.normal(0, 0.3, (200, 2 * 12)).astype(np.float32)     # 2 classes x T=3
    out['xformT_boxes'], out['xformT_deltas'] = tboxes, tdeltas
    out['xformT_out'] = rbox.bbox_transform(tboxes, tdeltas, (10., 10., 5., 5.))

    # ---- GenerateProposals (2-D level and T=3 tubes) ---------------------------
    from ops.generate_proposals import GenerateProposalsOp
    cfg.TEST.RPN_PRE_NMS_TOP_N = 1000
    cfg.TEST.RPN_POST_NMS_TOP_N = 300
    cfg.TEST.RPN_NMS_THRESH = 0.7
    for name, T, A, H, W, stride, anchors in [
            ('gp2d', 1, 3, 25, 42, 32, out['anchors_fpn5']),
            ('gp3d', 3, 12, 13, 21, 16, out['anchors_rpn12_T3'])]:
        scores = rng.permutation(A * H * W).reshape(1, A, H, W).astype(np.float32) / (A * H * W)
        deltas = rng.normal(0, 0.4, (1, 4 * A * T, H, W)).astype(np.float32)
        im_info = np.array([[H * stride, W * stride, 1.25]], dtype=np.float32)
        op = GenerateProposalsOp(anchors, 1. / stride, False)
        o = [Blob(), Blob()]
        op.forward([Blob(scores), Blob(deltas), Blob(im_info)], o)
        out[name + '_scores'], out[name + '_deltas'], out[name + '_im_info'] = scores, deltas, im_info
        out[name + '_rois'], out[name + '_probs'] = o[0].data, o[1].data
        out[name + '_stride'] = np.array(stride)

    # ---- collect / distribute / map_rois_to_fpn_levels -------------------------
    src = open(os.path.join(REF, 'modeling', 'FPN.py')).read()
    start = src.index('def map_rois_to_fpn_levels'); end = src.index('def add_multilevel_roi_blobs')
    ns = {'np': np, 'box_utils': rbox, 'cfg': cfg}
    exec(src[start:end], ns)
    fpn_stub = types.ModuleType('modeling.FPN')
    fpn_stub.map_rois_to_fpn_levels = ns['map_rois_to_fpn_levels']
    import modeling
    sys.modules['modeling.FPN'] = fpn_stub
    modeling.FPN = fpn_stub
    for name in ['datasets', 'datasets.json_dataset', 'roi_data', 'roi_data.fast_rcnn', 'utils.blob']:
        if name not in sys.modules:
            sys.modules[name] = types.ModuleType(name)
    sys.modules['utils.blob'].py_op_copy_blob = lambda src_arr, blob: setattr(blob, 'data', np.array(src_arr))
    import importlib
    cd = importlib.import_module('ops.collect_and_distribute_fpn_rpn_proposals')
    cfg.TEST.RPN_POST_NMS_TOP_N = 1000
    for name, T in [('cd2d', 1), ('cd3d', 3)]:
        rois_l, sc_l = [], []
        for lvl in range(2, 7):
            n = int(rng.integers(50, 400))
            smax = 40 * 2 ** (lvl - 1)
            t = rand_tubes(rng, n, T, smin=4, smax=smax)
            rois_l.append(np.hstack([np.zeros((n, 1), np.float32), t]).astype(np.float32))
            sc_l.append(rng.random((n, 1)).astype(np.float32))
        allsc = np.concatenate(sc_l).ravel()
        assert len(np.unique(allsc)) == len(allsc)
        rois = cd.collect([Blob(r) for r in rois_l] + [Blob(s) for s in sc_l], False)
        outs = [Blob() for _ in range(6)]
        cd.distribute(rois, None, outs, False)
        for i, r in enumerate(rois_l):
            out['%s_in_rois%d' % (name, i)] = r
            out['%s_in_scores%d' % (name, i)] = sc_l[i]
        out[name + '_rois'] = outs[0].data
        for i in range(4):
            out['%s_rois_fpn%d' % (name, i + 2)] = outs[1 + i].data
        out[name + '_idx_restore'] = outs[5].data
        out[name + '_lvls'] = ns['map_rois_to_fpn_levels'](rois[:, 1:], 2, 5)

    # ---- RoIToBatchFormat ------------------------------------------------------
    src = open(os.path.join(REF, 'ops', 'roi_blob_transforms.py')).read()
    ns2 = {'np': np}
    exec(src[src.index('class RoIToBatchFormatOp'):], ns2)
    tub = np.hstack([rng.integers(0, 2, (40, 1)).astype(np.float32), rand_tubes(rng, 40, 3)]).astype(np.float32)
    o = [Blob()]
    ns2['RoIToBatchFormatOp']().forward([Blob(tub)], o)
    out['r2b_in'], out['r2b_out'] = tub, o[0].data

    # ---- scipy LSA (installed scipy == what tracking_engine.py:237 would call here)
    import scipy.optimize
    from oracle.tracking import synth_video, distance_matrix
    frames = synth_video(np.random.default_rng(3), n_frames=6, n_dets=100)
    for i in range(1, 6):
        C = distance_matrix(frames[i - 1], frames[i])
        r, c = scipy.optimize.linear_sum_assignment(C)
        out['lsa_C%d' % i], out['lsa_r%d' % i], out['lsa_c%d' % i] = C, r, c
    Cr = np.ones((37, 61), np.float32); m = rng.random(Cr.shape) < 0.1; Cr[m] = rng.random(int(m.sum()))
    for nm, C in [('wide', Cr), ('tall', Cr.T.copy())]:
        r, c = scipy.optimize.linear_sum_assignment(C)
        out['lsa_C_' + nm], out['lsa_r_' + nm], out['lsa_c_' + nm] = C, r, c

    # the compiled reference Cython itself on the seeded inputs of tests/test_oracle_boxes.py (*_vs_compiled_reference)
    from oracle._ref import cython_bbox, cython_nms
    rng = np.random.default_rng(5)
    for i, scale in enumerate((0.02, 1.0, 7.0)):
        x1 = rng.uniform(0, 500, 400); y1 = rng.uniform(0, 300, 400)
        a = np.stack([x1, y1, x1 + rng.uniform(0, 200, 400) * scale, y1 + rng.uniform(0, 200, 400) * scale], 1).astype(np.float32)
        out['refcy_iou_boxes_%d' % i], out['refcy_iou_out_%d' % i] = a, cython_bbox.bbox_overlaps(a[:250], a[250:])
    rng = np.random.default_rng(7)
    c = rng.uniform(0, 600, (60, 2))
    xy = c[rng.integers(0, 60, 1500)] + rng.normal(0, 12, (1500, 2))
    wh = rng.uniform(20, 120, (1500, 2))
    d = np.hstack([xy, xy + wh, rng.permutation(1500)[:, None] / 1500.]).astype(np.float32)
    out['refcy_nms_dets'] = d
    for th in (0.3, 0.7):
        out['refcy_nms_keep_%d' % int(th * 10)] = np.asarray(cython_nms.nms(d, np.float32(th)), dtype=np.int64)

    groups = {}
    for k, v in out.items():
        groups.setdefault(k.split('_')[0], {})[k] = np.asarray(v)
    for g, d in groups.items():
        np.savez_compressed(os.path.join(HERE, g + '.npz'), **d)
        print(g, sum(v.nbytes for v in d.values()) // 1024, 'KiB')


if __name__ == '__main__':
    main()
