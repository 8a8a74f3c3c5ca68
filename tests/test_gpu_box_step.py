"""GPU: every launch key of the box stages on the benchmarked steps (dt_rpn_proposals_multi, dt_nms_batched, dt_collect_rpn,
dt_distribute_fpn, dt_box_decode, dt_limit_detections, dt_rpn_targets, dt_sample_rois), launched at the step's shapes and
compared exactly with the host references of tests/test_box_reference.py and oracle/, plus a coverage test that proves the table
lists every key DetectionEngine.detect (r50fpn3d, r50fpn2d, r18tube, every dtype the engine takes) and KeypointRcnnTrainer.step
launch, and a teacher-forced capture of the real steps whose downstream stages are re-run by the oracle on the device's own
upstream output.

Selection, order, counts, keep lists, levels, restore indices and labels are asserted equal.  The only inexact steps are
expf (2-D decode and softmax score: compared as membership in the derived candidate sets of test_box_reference) and the
two log columns of the box targets (8 ulp, as tests/test_gpu_targets.py)."""
import inspect

import numpy as np
import pytest
import torch

from oracle import boxes as obox
from oracle import proposals as oprop
from oracle import targets as ot
from test_box_reference import (F32, F64, clip_boxes, decode2d_set, grid_logits, limit_ref, match_rows, rank_keys,
                                rpn_ref, score_filter_state, softmax_candidates, time_mean)

pytestmark = pytest.mark.gpu

GE, GT = 0, 1                    # box_ops.NMS_2D_GE, NMS_TUBE_GT
BY_SCORE, BY_INDEX = 0, 1        # box_ops.ORDER_SCORE, ORDER_INDEX
FPN5 = ((200, 336), (100, 168), (50, 84), (25, 42), (13, 21))     # P2..P6 of the 800 x 1344 blob
TUBE = ((50, 84),)                                                  # R18 conv4 of the 800 x 1334 blob
A_FPN, A_TUBE = 3, 12
TUBE_SIZES = (64, 128, 256, 512)

# ------------------------------------------------------------------ the launch table
# dt_rpn_proposals_multi: (level shapes, A, T, act_f32, pre_nms_topn, min_size > 0, time_major)
RPN = {(FPN5, A_FPN, 1, 1, 1000, False, False),          # FPN inference, all levels in one launch
       (FPN5, A_FPN, 1, 1, 2000, False, False),          # FPN training proposals
       (TUBE, A_TUBE, 3, 1, 1000, False, True)}          # r18tube: time-major tube RPN
# dt_nms_batched: (nmax, T, cmp_mode, out_order, max_keep, thresh, counts given)
NMS = {(1000, 1, GE, BY_INDEX, 1000, 0.7, True), (1000, 1, GE, BY_INDEX, 0, 0.5, True),
       (2000, 1, GE, BY_INDEX, 2000, 0.7, True),
       (1000, 3, GT, BY_SCORE, 1000, 0.7, True), (1000, 3, GT, BY_SCORE, 0, 0.5, True)}
# dt_collect_rpn: (L, K, T, post_nms_topn, R)
COLLECT = {(5, 1000, 1, 1000, 1000), (5, 2000, 1, 2000, 2000), (1, 1000, 3, 1000, 1000)}
# dt_distribute_fpn: (ld, col0, T, k_min, k_max, n_dev given, restore wanted)
DISTRIBUTE = {(5, 1, 1, 2, 5, False, False)}
# dt_box_decode: (T, num_classes, ld_c > C, score_thresh)
BOX_DECODE = {(1, 2, True, 0.05), (3, 2, False, 0.05)}
# dt_limit_detections: (num_classes, R, T, max_per_im, cap)
LIMIT = {(2, 1000, 1, 100, 104), (2, 1000, 3, 100, 104)}
# dt_rpn_targets: (levels, A, T, batch, fg_fraction, straddle)
RPN_TARGETS = {(FPN5, A_FPN, 1, 256, 0.5, 0.0)}
# dt_sample_rois: (R, topn, T, K, batch, Gmax)
SAMPLE = {(2000, 2000, 1, 17, 512, 8)}
TABLE = dict(dt_rpn_proposals_multi=RPN, dt_nms_batched=NMS, dt_collect_rpn=COLLECT, dt_distribute_fpn=DISTRIBUTE,
             dt_box_decode=BOX_DECODE, dt_limit_detections=LIMIT, dt_rpn_targets=RPN_TARGETS, dt_sample_rois=SAMPLE)


def launch_key(name, a):
    """The table key of one L.call(name, *a) of these entry points, or None for other entry points."""
    if name == 'dt_rpn_proposals_multi':
        return (tuple((a[0][i].H, a[0][i].W) for i in range(a[1])), a[4], a[5], a[2], a[7], a[8] > 0, bool(a[12]))
    if name == 'dt_nms_batched':
        return (a[2], a[4], a[7], a[8], a[9], round(a[6], 4), a[5] is not None)
    if name == 'dt_collect_rpn':
        return (a[4], a[5], a[6], a[7], a[11])
    if name == 'dt_distribute_fpn':
        return (a[3], a[4], a[5], a[6], a[7], a[2] is not None, a[11] is not None)
    if name == 'dt_box_decode':
        return (a[4], a[9], a[6] > a[9], round(a[14], 4))
    if name == 'dt_limit_detections':
        return (a[4], a[5], a[6], a[7], a[10])
    if name == 'dt_rpn_targets':
        return (tuple((a[0][i].H, a[0][i].W) for i in range(a[1])), a[2], a[3], a[13], round(a[14], 4), round(a[10], 4))
    if name == 'dt_sample_rois':
        return (a[4], a[5], a[13], a[12], a[16], a[11])
    return None


def _train_cfg():
    import bench
    cfg = bench.bench_cfg(800, 1333, 'r50fpn3d')
    cfg.TRAIN.BATCH_SIZE_PER_IM = 512; cfg.TRAIN.RPN_PRE_NMS_TOP_N = 2000
    return cfg


def test_step_box_ops_are_all_in_the_table(record_property):
    """One 800 x 1333 clip of each bench workload through DetectionEngine.detect in bf16, bf16x3, bf16x3h and tf32x3 (where
    the engine takes them), and one KeypointRcnnTrainer.step at the bench training config: every launch of the box entry
    points has a key in TABLE, each of which has a value test below."""
    import step_launches as sl
    missing, seen = {}, set()
    for run in [(wl, m) for wl in sl.WORKLOADS for m in ('bf16', 'bf16x3', 'bf16x3h', 'tf32x3')] + ['train']:
        rec = sl.record(run)
        if not rec.taken:
            assert run[1] not in ('bf16', 'bf16x3'), run
            continue
        launched = [(name, k) for name, a, _ in rec.calls if (k := launch_key(name, a)) is not None]
        names = {n for n, _ in launched}
        if run == 'train':
            assert {'dt_rpn_targets', 'dt_sample_rois'} <= names
        else:
            assert {'dt_rpn_proposals_multi', 'dt_nms_batched', 'dt_collect_rpn', 'dt_box_decode', 'dt_limit_detections'} <= names
        for name, k in launched:
            seen.add((name, k))
            if k not in TABLE[name]:
                missing.setdefault((name, k), run)
    record_property('keys_seen', len(seen))
    print('box keys seen: %d' % len(seen))
    for s in sorted(seen, key=str):
        print('  ', s)
    assert not missing, missing


# ------------------------------------------------------------------ RPN proposals
def _cell_anchors(T):
    if T == 1:
        return [oprop.generate_anchors(2. ** l, (32 * 2. ** (l - 2),), (0.5, 1, 2)) for l in range(2, 7)]
    return [oprop.generate_anchors(16, TUBE_SIZES, (0.5, 1, 2), T)]


def _rpn_inputs(T, A, shapes, seed, pick=None):
    """Per level the engine's RPN output layout: fp32 [B, H, W, ld] (time-major: [B, T, H, W, ld]) with the logits in the
    first A channels, the deltas in the next 4A and a poison column after them.  Grid logits (test_box_reference); per
    image: 0, 5..7 plain grid; 1 a K-th key shared by far more anchors than needed, spread over every slice; 2 a fully flat
    map; 3 saturated anchors (>= 17 in every frame, score exactly 1.0), on P2 more of them than K; 4 deltas past
    BBOX_XFORM_CLIP and boxes decoded wholly outside the image.  `pick` selects images of the 8."""
    rng = np.random.default_rng(seed)
    ld = (5 * A + 3) // 4 * 4
    B = 8
    outs = []
    for (H, W) in shapes:
        lead = (B, T) if T > 1 else (B,)
        o = np.full(lead + (H, W, ld), 999.0, F32)
        lg = grid_logits(rng, lead + (H, W, A))
        lg[1] = rng.choice(np.array([-0.5, 0.0, 0.125], F32), size=lg[1].shape, p=[0.6, 0.39, 0.01])
        lg[2] = F32(0.25)
        sat = rng.random((H, W, A)) < 0.06
        lg[3][..., sat] = rng.choice(np.array([17.0, 20.0, 30.0], F32), size=lg[3][..., sat].shape)
        dl = rng.normal(0, 0.3, lead + (H, W, 4 * A)).astype(F32)
        far = rng.random(dl[4].shape) < 0.2
        dl[4][far] = rng.uniform(4.2, 12.0, int(far.sum())).astype(F32) * np.sign(rng.normal(size=int(far.sum()))).astype(F32)
        out = rng.random(dl[4].shape[:-1] + (A,)) < 0.1
        d4 = dl[4].reshape(dl[4].shape[:-1] + (A, 4))
        d4[..., 0][out] = rng.uniform(50, 200, int(out.sum())).astype(F32) * rng.choice(np.array([-1, 1], F32), int(out.sum()))
        dl[4] = d4.reshape(dl[4].shape)
        o[..., :A] = lg
        o[..., A:5 * A] = dl
        outs.append(o if pick is None else np.ascontiguousarray(o[list(pick)]))
    return outs


def _launch_rpn(outs, anchors, im_info, K, min_size, T, A, time_major):
    from detectandtrack_b200 import _lib as L
    from detectandtrack_b200.ops import rpn_ops
    B = outs[0].shape[0]
    Lv = len(outs)
    Kb = max(min(K, o.shape[-3] * o.shape[-2] * A) for o in outs)
    props = L.zeros((B, Lv, Kb, 4 * T + 1), torch.float32)
    counts = L.zeros((B, Lv), torch.int32)
    props.fill_(-5.0)
    levels = []
    for l, o in enumerate(outs):
        od = torch.from_numpy(o).cuda()
        levels.append(dict(logits=od[..., :A], deltas=od[..., A:5 * A], anchors=anchors[l], feat_stride=2. ** (l + 2) if T == 1 else 16.,
                           out=props[:, l], counts=counts[:, l]))
    rpn_ops.rpn_proposals_levels(levels, torch.from_numpy(im_info).cuda(), K, A, min_size, T, time_major=time_major)
    return props.cpu().numpy(), counts.cpu().numpy()


def _check_rpn(outs, props, counts, cells, im_info, K, min_size, T, A, rec):
    """Every (image, level) against rpn_ref: selection, order, count and score column exact; boxes bit-exact for tubes and
    among the 2-D candidates.  The expected score of an anchor is the kernel's formula in fp32 on the device (torch's fp32
    exp is the same correctly-rounded-to-2-ulp expf; equal inputs give equal bits), 1 / (1 + exp(-x))."""
    und = []
    for l, o in enumerate(outs):
        H, W = o.shape[-3:-1]
        stride = 2. ** (l + 2) if T == 1 else 16.
        anchors = oprop.shifted_anchors(cells[l], H, W, stride, T)
        for b in range(o.shape[0]):
            if T == 1:
                x = o[b, :, :, :A].reshape(-1)
                dl = o[b, :, :, A:5 * A].reshape(-1, 4)
            else:
                x = time_mean(o[b, :, :, :, :A].reshape(T, -1))
                dl = o[b, :, :, :, A:5 * A].reshape(T, H * W, A, 4).transpose(1, 2, 0, 3).reshape(-1, 4 * T)
            ref = rpn_ref(rank_keys(x), dl, anchors, im_info[b], K, min_size, T)
            xs = torch.from_numpy(o[b][..., :A].reshape((T, -1) if T > 1 else (-1,))).cuda()
            if T > 1:
                acc = xs[0]
                for t in range(1, T):
                    acc = acc + xs[t]
                xs = acc / float(T)
            sc = (1.0 / (1.0 + torch.exp(-xs))).cpu().numpy()[ref['idx']]
            n = int(counts[b, l])
            und.append(match_rows(props[b, l, :n], ref, sc))
            assert (props[b, l, n:] == -5.0).all(), (b, l)          # nothing written past the count
    rec('undecided_2d_rows', int(sum(und)))


RPN_VALUE_KEYS = sorted(RPN, key=str) + [(FPN5, A_FPN, 1, 1, 1000, True, False), (TUBE, A_TUBE, 3, 1, 1000, True, True)]


@pytest.mark.parametrize('key', RPN_VALUE_KEYS, ids=lambda k: 'L%d-T%d-K%d-min%d' % (len(k[0]), k[2], k[4], k[5]))
def test_rpn_proposals_step_shape_exact(key, record_property):
    """dt_rpn_proposals_multi as the steps launch it: all levels of a B-clip batch (B = 8 inference, 2 training) in one launch
    into strided props[:, l] / counts[:, l], grid logits with the crafted images of _rpn_inputs.  Then per-image independence:
    image b launched alone is bit-identical, and permuting the images permutes the output."""
    shapes, A, T, _, K, has_min, tm = key
    B = 2 if K == 2000 else 8                                           # training: the shared K-th key and the saturated image
    min_size = 16.0 if has_min else 0.0
    outs = _rpn_inputs(T, A, shapes, seed=K + T + has_min, pick=(1, 3) if B == 2 else None)
    cells = _cell_anchors(T)
    anchors = [torch.from_numpy(np.ascontiguousarray(c, F64)).cuda() for c in cells]
    H0, W0 = shapes[0]
    im_info = np.array([[H0 * (4 if T == 1 else 16), W0 * (4 if T == 1 else 16) - 11, 1.0]] * B, F32)
    im_info[1, 2] = 1.25                                                # per-image scale: min_size * scale
    props, counts = _launch_rpn(outs, anchors, im_info, K, min_size, T, A, tm)
    _check_rpn(outs, props, counts, cells, im_info, K, min_size, T, A, record_property)
    for b in (0, B - 1):
        p1, c1 = _launch_rpn([o[b:b + 1] for o in outs], anchors, im_info[b:b + 1], K, min_size, T, A, tm)
        assert np.array_equal(c1[0], counts[b]) and np.array_equal(p1[0], props[b]), b
    perm = np.random.default_rng(0).permutation(B)
    pp, cp = _launch_rpn([np.ascontiguousarray(o[perm]) for o in outs], anchors, im_info[perm], K, min_size, T, A, tm)
    assert np.array_equal(cp, counts[perm]) and np.array_equal(pp, props[perm])


# ------------------------------------------------------------------ NMS
def nms_ref(rows, thresh, cmp_mode, out_order, max_keep):
    """The keep list of one problem: nms_2d ('>=') or nms_tubes ('>'), in ascending index or score order (descending score,
    then descending index: the oracle's score_order), then keep[:max_keep] as generate_proposals.py:108-110 applies it."""
    if len(rows) == 0:
        return np.zeros(0, np.int64)
    k = obox.nms_2d(rows, thresh) if cmp_mode == GE else np.array(obox.nms_tubes(rows, thresh))
    if out_order == BY_INDEX:
        k = np.sort(k)
    else:
        s = set(int(i) for i in k)
        k = np.array([i for i in obox.score_order(rows[:, -1]) if int(i) in s])
    return k[:max_keep] if max_keep > 0 else k


def check_nms(dets, counts, thresh, cmp_mode, out_order, max_keep, keep, num):
    nmax = dets.shape[1]
    for p in range(dets.shape[0]):
        n = min(int(counts[p]), nmax) if counts is not None else nmax
        k = nms_ref(dets[p, :n], thresh, cmp_mode, out_order, max_keep)
        assert int(num[p]) == len(k) and np.array_equal(keep[p, :len(k)], k), (p, int(num[p]), len(k))


def _nms_problems(P, nmax, T, seed):
    """P problems of nmax rows (score-descending like the RPN's props, ragged counts with an empty problem and a full one):
    clusters of jittered boxes, so IoU lands on both sides of the threshold, and scores on a coarse grid, so exact ties occur."""
    rng = np.random.default_rng(seed)
    d = np.zeros((P, nmax, 4 * T + 1), F32)
    for p in range(P):
        c = rng.uniform(0, 1200, (40, 2))
        ci = rng.integers(0, 40, nmax)
        wh = rng.uniform(20, 300, (40, 2))[ci] * rng.uniform(0.8, 1.25, (nmax, 2))
        for t in range(T):
            ctr = c[ci] + rng.normal(0, 12, (nmax, 2)) + 5 * t
            d[p, :, 4 * t:4 * t + 4] = np.concatenate([ctr - wh / 2, ctr + wh / 2], 1)
        d[p, :, -1] = np.sort(np.round(rng.uniform(0, 1, nmax) * 64) / 64)[::-1]
    counts = rng.integers(0, nmax + 1, P).astype(np.int32)
    counts[0], counts[-1] = 0, nmax
    return d, counts


NMS_VALUE_KEYS = sorted(NMS) + [(1000, 1, GE, BY_SCORE, 300, 0.7, True), (1000, 1, GT, BY_INDEX, 0, 0.5, True),
                                (1000, 3, GT, BY_INDEX, 1000, 0.7, True), (1000, 1, GT, BY_SCORE, 0, 0.7, False)]


@pytest.mark.parametrize('key', NMS_VALUE_KEYS, ids=lambda k: '-'.join(str(v) for v in k))
def test_nms_step_shape_exact(key):
    """dt_nms_batched at the steps' problem shapes (40 x 1000 FPN RPN levels, 8 x 1000 box-head classes, 10 x 2000 training
    levels, 8 x 1000 tube problems) with ragged counts, an empty problem and tied scores, both comparators and both output
    orders: keep lists equal oracle.boxes.nms's; permuting the problems permutes the output."""
    from detectandtrack_b200.ops import box_ops
    nmax, T, cmp_mode, order, max_keep, thresh, has_counts = key
    P = {1000: 40 if max_keep else 8, 2000: 10}[nmax]
    dets, counts = _nms_problems(P, nmax, T, seed=nmax + T + cmp_mode + order)
    cnt = torch.from_numpy(counts).cuda() if has_counts else None
    keep, num = box_ops.nms_batched(torch.from_numpy(dets).cuda(), cnt, thresh, cmp_mode, order, max_keep=max_keep)
    keep, num = keep.cpu().numpy(), num.cpu().numpy()
    check_nms(dets, counts if has_counts else None, thresh, cmp_mode, order, max_keep, keep, num)
    perm = np.random.default_rng(1).permutation(P)
    k2, n2 = box_ops.nms_batched(torch.from_numpy(np.ascontiguousarray(dets[perm])).cuda(),
                                 torch.from_numpy(counts[perm]).cuda() if has_counts else None, thresh, cmp_mode, order, max_keep=max_keep)
    n2 = n2.cpu().numpy()
    assert np.array_equal(n2, num[perm])
    k2 = k2.cpu().numpy()
    for i, p in enumerate(perm):
        assert np.array_equal(k2[i, :n2[i]], keep[p, :num[p]])


# ------------------------------------------------------------------ collect / distribute
def check_collect(props, keep, nkeep, post, R, rois, scores, counts):
    """Per image: oracle.proposals.collect over the levels' kept rows (np.argsort(-score) stable: ties to the earlier level,
    then the earlier keep position), cut at post_nms_topn and R."""
    B, L, K, ld = props.shape
    for b in range(B):
        rl, sl = [], []
        for l in range(L):
            rows = props[b, l, keep[b * L + l, :min(int(nkeep[b * L + l]), K)]]
            rl.append(np.hstack([np.full((len(rows), 1), b, F32), rows[:, :-1]]))
            sl.append(rows[:, -1:])
        sc = np.concatenate(sl)[:, 0]
        cut = min(post if post > 0 else len(sc), R)
        ref = oprop.collect(rl, sl, cut) if len(sc) else np.zeros((0, ld), F32)
        inds = np.argsort(-sc, kind='stable')[:cut]
        n = len(ref)
        assert int(counts[b]) == n, (b, int(counts[b]), n)
        assert np.array_equal(rois[b, :n], ref) and np.array_equal(scores[b, :n], sc[inds]), b


COLLECT_VALUE_KEYS = sorted(COLLECT) + [(5, 1000, 1, 700, 1000), (5, 2000, 1, 0, 10000)]


@pytest.mark.parametrize('key', COLLECT_VALUE_KEYS, ids=lambda k: '-'.join(map(str, k)))
def test_collect_step_shape_exact(key):
    """dt_collect_rpn at L*K = 5000 and 10 000 (the largest shared-memory sorts) and the tube's single level: keep lists in
    ascending row order with ragged counts, an empty level, and scores on a coarse grid shared across levels (cross-level
    ties); permuting the images permutes the output."""
    from detectandtrack_b200.ops import rpn_ops
    L, K, T, post, R = key
    B = 2 if K == 2000 else 8
    rng = np.random.default_rng(L * K + post)
    props = np.zeros((B, L, K, 4 * T + 1), F32)
    props[..., :4 * T] = rng.uniform(0, 1300, props[..., :4 * T].shape)
    props[..., -1] = np.sort(np.round(rng.uniform(0, 1, (B, L, K)) * 256) / 256, -1)[..., ::-1]
    nkeep = rng.integers(0, K + 1, B * L).astype(np.int32)
    nkeep[1] = 0
    nkeep[0] = K
    keep = np.zeros((B * L, K), np.int32)
    for p in range(B * L):
        keep[p, :nkeep[p]] = np.sort(rng.choice(K, nkeep[p], replace=False))
    rois, scores, counts = rpn_ops.collect(torch.from_numpy(props).cuda(), torch.from_numpy(keep).cuda(), torch.from_numpy(nkeep).cuda(), post, R)
    rois, scores, counts = rois.cpu().numpy(), scores.cpu().numpy(), counts.cpu().numpy()
    check_collect(props, keep, nkeep, post, R, rois, scores, counts)
    perm = np.random.default_rng(2).permutation(B)
    kp = keep.reshape(B, L, K)[perm].reshape(B * L, K)
    r2, s2, c2 = rpn_ops.collect(torch.from_numpy(np.ascontiguousarray(props[perm])).cuda(), torch.from_numpy(np.ascontiguousarray(kp)).cuda(),
                                 torch.from_numpy(np.ascontiguousarray(nkeep.reshape(B, L)[perm].reshape(-1))).cuda(), post, R)
    c2 = c2.cpu().numpy()
    assert np.array_equal(c2, counts[perm]) and np.array_equal(s2.cpu().numpy(), scores[perm])
    r2 = r2.cpu().numpy()
    assert np.array_equal(r2[..., 1:], rois[perm][..., 1:])
    for i in range(B):
        assert (r2[i, :c2[i], 0] == i).all()


def check_distribute(rois, n, col0, T, kmin, kmax, s0, lvl0, levels, restore):
    r = rois[:n, col0:col0 + 4 * T]
    lv = oprop.map_rois_to_fpn_levels(r, kmin, kmax, s0, lvl0).astype(np.int64)
    assert np.array_equal(levels[:n], lv)
    if restore is not None:
        order = np.concatenate([np.where(lv == l)[0] for l in range(kmin, kmax + 1)])
        assert np.array_equal(restore[:n], np.argsort(order, kind='stable'))


DISTRIBUTE_VALUE_KEYS = sorted(DISTRIBUTE) + [(5, 1, 1, 2, 5, True, True), (5, 1, 1, 2, 5, False, True)]


@pytest.mark.parametrize('key', DISTRIBUTE_VALUE_KEYS, ids=lambda k: '-'.join(str(int(v)) for v in k))
def test_distribute_step_shape_exact(key):
    """dt_distribute_fpn over one CTA's B*R = 8000 rows: collect-like random boxes, zero padding rows, and squares whose
    sqrt(area) is one ulp either side of 112, 224 and 448 (the level boundaries): levels and restore index equal
    map_rois_to_fpn_levels / distribute's."""
    from detectandtrack_b200.ops import rpn_ops
    ld, col0, T, kmin, kmax, has_ndev, want_restore = key
    rng = np.random.default_rng(5)
    n = 8000
    rois = np.zeros((n, ld), F32)
    x1, y1 = rng.uniform(0, 1000, n), rng.uniform(0, 700, n)
    w, h = np.exp(rng.uniform(0, np.log(900), n)), np.exp(rng.uniform(0, np.log(700), n))
    rois[:, 1:5] = np.stack([x1, y1, x1 + w, y1 + h], 1)
    rois[:, 0] = np.arange(n) // 1000
    i = 0
    for s in (112.0, 224.0, 448.0):
        for side in (F32(s), np.nextafter(F32(s), F32(0)), np.nextafter(F32(s), F32(1e9)),
                     np.nextafter(np.nextafter(F32(s), F32(0)), F32(0))):
            for x0 in (0.0, 3.5, 517.25):
                rois[i, 1:5] = [x0, x0, F32(x0) + side - F32(1), F32(x0) + side - F32(1)]
                i += 1
    pad = rng.random(n) < 0.1
    pad[:i] = False
    rois[pad] = 0.0
    nd = n - 321 if has_ndev else n
    lv, restore, lc = rpn_ops.distribute(torch.from_numpy(rois).cuda(), torch.tensor([nd], dtype=torch.int32).cuda() if has_ndev else None,
                                         col0=col0, T=T, k_min=kmin, k_max=kmax, want_restore=want_restore)
    check_distribute(rois, nd, col0, T, kmin, kmax, 224.0, 4.0, lv.cpu().numpy(), restore.cpu().numpy() if want_restore else None)
    levels_crafted = lv[:i].cpu().numpy()
    assert len(set(levels_crafted.tolist())) >= 3                      # the crafted squares do land on several levels


# ------------------------------------------------------------------ box decode / limit
def check_box_decode(rois, roi_counts, cls, bbox, C, im_info, im_hw, weights, thresh, T, dets, cnt):
    """Per (image, class j >= 1): the rows i < roi_counts whose score passes '> thresh', in row order.  A row is kept when
    every softmax candidate passes, absent when none does, and otherwise (inside the band) kept exactly when the device
    score, itself one of the candidates, is > thresh.  Boxes: the 2-D candidates / the fp64 tube decode bit-exact, clipped
    to the original image.  Returns the number of rows inside the score band."""
    B, R, _ = rois.shape
    band = 0
    for b in range(B):
        n = min(int(roi_counts[b]), R)
        rows = slice(b * R, b * R + n)
        boxes = (rois[b, :n, 1:] / F32(im_info[b, 2])).astype(F32)
        for j in range(1, C):
            d = bbox[rows, j * 4 * T:(j + 1) * 4 * T]
            cand = decode2d_set(boxes, d, weights, obox.BBOX_XFORM_CLIP) if T == 1 else obox.bbox_transform(boxes, d, weights)[None]
            cand = clip_boxes(cand, im_hw[b, 0], im_hw[b, 1])
            sc = softmax_candidates(cls[rows, :C], j)
            st = score_filter_state(sc, thresh)
            got = dets[b, j - 1, :int(cnt[b * (C - 1) + j - 1])]
            r = 0
            for i in range(n):
                if st[i] == 0:
                    continue
                hit = r < len(got) and bool((got[r, :-1][None] == cand[:, i]).any(0).all()) and bool((got[r, -1] == sc[:, i]).any())
                if st[i] == -1:
                    band += 1
                    if not (hit and got[r, -1] > F32(thresh)):
                        continue
                assert hit, (b, j, i, r)
                r += 1
            assert r == len(got), (b, j, r, len(got))
            assert (got[:, -1] > F32(thresh)).all()
    return band


BOX_VALUE_KEYS = sorted(BOX_DECODE) + [(1, 2, False, 0.05), (3, 2, True, 0.05)]


@pytest.mark.parametrize('key', BOX_VALUE_KEYS, ids=lambda k: 'T%d-C%d-ld%d' % k[:3])
def test_box_decode_step_shape(key, record_property):
    """dt_box_decode on 8 clips x 1000 RoIs (roi_counts < R on some), logits / deltas as strided column slices of the
    cls_bbox output (2-D) or the contiguous fold_tube_heads output (tubes), scores placed within a few ulp of 0.05 on both
    sides, deltas past the clip; permuting the images permutes the output."""
    from detectandtrack_b200.ops import rpn_ops
    T, C, strided, thresh = key
    B, R = 8, 1000
    rng = np.random.default_rng(T + 2 * strided)
    rois = np.zeros((B, R, 4 * T + 1), F32)
    rois[:, :, 0] = np.arange(B)[:, None]
    x1, y1 = rng.uniform(0, 1200, (B, R)), rng.uniform(0, 700, (B, R))
    w, h = rng.uniform(1, 400, (B, R)), rng.uniform(1, 400, (B, R))
    for t in range(T):
        rois[:, :, 1 + 4 * t:5 + 4 * t] = np.stack([x1 + t, y1, x1 + w + t, y1 + h], -1)
    counts = np.array([R, 0, 999, 1, 500, R, 64, 777], np.int32)
    ld = (C + 4 * T * C + 3) // 4 * 4 + (4 if T > 1 else 0)            # 12: the engine's cls_bbox_ld for C = 2
    logits = rng.normal(0, 2, (B * R, C)).astype(F32)
    # on the threshold: l1 - l0 = log(0.05 / 0.95) plus a few ulps of l1
    edge = rng.random(B * R) < 0.3
    l0 = logits[edge, 0]
    l1 = (l0.astype(F64) + np.log(0.05 / 0.95)).astype(F32)
    steps = rng.integers(-4, 5, int(edge.sum()))
    for k in range(int(edge.sum())):
        for _ in range(abs(steps[k])):
            l1[k] = np.nextafter(l1[k], F32(np.inf) if steps[k] > 0 else F32(-np.inf))
    logits[edge, 1] = l1
    deltas = rng.normal(0, 1.0, (B * R, 4 * T * C)).astype(F32)
    deltas[::9, 2::4] = 6.0
    if strided:
        o = np.full((B * R, ld), 777.0, F32)
        o[:, :C] = logits
        o[:, C:C + 4 * T * C] = deltas
        od = torch.from_numpy(o).cuda()
        cls_d, bbox_d = od[:, :C], od[:, C:C + 4 * T * C]
    else:
        cls_d, bbox_d = torch.from_numpy(logits).cuda(), torch.from_numpy(deltas).cuda()
    im_info = np.array([[800, 1344, 1.0]] * B, F32)
    im_info[3, 2] = 1.5
    im_hw = np.array([[800, 1333]] * B, F32)
    im_hw[3] = [533, 889]
    w4 = (10., 10., 5., 5.)
    run = lambda r, c, cl, bb, ii, hw: rpn_ops.box_decode(torch.from_numpy(np.ascontiguousarray(r)).cuda(), torch.from_numpy(c).cuda(), cl, bb, C,
                                                          torch.from_numpy(np.ascontiguousarray(ii)).cuda(),
                                                          torch.from_numpy(np.ascontiguousarray(hw)).cuda(), w4, thresh, T)
    dets, cnt = run(rois, counts, cls_d, bbox_d, im_info, im_hw)
    dets, cnt = dets.cpu().numpy(), cnt.cpu().numpy()
    band = check_box_decode(rois, counts, logits, deltas, C, im_info, im_hw, w4, thresh, T, dets, cnt)
    record_property('rows_in_score_band', band)
    assert band > 0
    perm = np.random.default_rng(3).permutation(B)
    rowperm = (perm[:, None] * R + np.arange(R)[None]).reshape(-1)
    cp, bp = cls_d[torch.from_numpy(rowperm).cuda()], bbox_d[torch.from_numpy(rowperm).cuda()]
    d2, c2 = run(rois[perm], counts[perm], cp, bp, im_info[perm], im_hw[perm])
    d2, c2 = d2.cpu().numpy(), c2.cpu().numpy()
    assert np.array_equal(c2, cnt.reshape(B, C - 1)[perm].reshape(-1))
    for i, p in enumerate(perm):
        n = c2[i]
        assert np.array_equal(d2[i, 0, :n], dets[p, 0, :n])


SENTINEL = -7777.0


def _launch_limit(dets, keep, nkeep, max_per_im, cap):
    """dt_limit_detections into a sentinel-filled buffer 64 rows larger than the B x (C-1) x cap slots."""
    from detectandtrack_b200 import _lib as L
    B, C1, R, ld = dets.shape
    T = (ld - 1) // 4
    out = torch.full(((B * C1 * cap + 64) * ld,), SENTINEL, dtype=torch.float32, device='cuda')
    cnt = L.zeros((B * C1,), torch.int32)
    dd, kd, nd = torch.from_numpy(dets).cuda(), torch.from_numpy(keep).cuda(), torch.from_numpy(nkeep).cuda()
    L.call('dt_limit_detections', L.ptr(dd), L.ptr(kd), L.ptr(nd), B, C1 + 1, R, T, int(max_per_im), L.ptr(out), L.ptr(cnt), cap, L.stream_ptr())
    o = out.cpu().numpy()
    return o[:B * C1 * cap * ld].reshape(B, C1, cap, ld), o[B * C1 * cap * ld:], cnt.cpu().numpy()


def check_limit(dets, keep, nkeep, max_per_im, cap, out, cnt):
    B, C1, R, ld = dets.shape
    for b in range(B):
        lists = [keep[b * C1 + c, :min(int(nkeep[b * C1 + c]), R)] for c in range(C1)]
        ref = limit_ref([dets[b, c, k, -1] for c, k in enumerate(lists)], max_per_im, cap)
        for c, (count, pos) in enumerate(ref):
            assert int(cnt[b * C1 + c]) == count, (b, c, int(cnt[b * C1 + c]), count)
            assert np.array_equal(out[b, c, :len(pos)], dets[b, c, lists[c][pos]]), (b, c)


@pytest.mark.parametrize('key', sorted(LIMIT), ids=lambda k: 'T%d' % k[2])
def test_limit_detections_ties_at_threshold(key):
    """dt_limit_detections with exactly 100, 101, 103, 105 and 109 rows at or above the 100th score (ties at it), fewer rows
    than the limit, and an empty keep list: out_counts is the full reference count, exactly the first cap rows are written
    (the rest of each slot block and the guard rows keep the sentinel); permuting the images permutes the output."""
    C, R, T, max_per_im, cap = key
    B, C1, ld = 8, C - 1, 4 * T + 1
    rng = np.random.default_rng(T)
    dets = np.zeros((B, C1, R, ld), F32)
    dets[..., :4 * T] = rng.uniform(0, 1000, (B, C1, R, 4 * T))
    keep = np.zeros((B * C1, R), np.int32)
    nkeep = np.zeros(B * C1, np.int32)
    tied = [1, 2, 4, 6, 10, 0, 0, 30]                        # rows at the threshold beyond the 99 distinct above it
    for b in range(B):
        nk = [300, 300, 300, 300, 300, 60, 0, 250][b]
        dets[b, 0, :, -1] = np.round(rng.uniform(0.06, 0.5, R) * 1e4) / 1e4
        sc = np.round(rng.uniform(0.06, 0.5, nk) * 1e4) / 1e4      # the kept rows' scores, below the threshold ...
        if tied[b]:
            sc[:99] = np.linspace(0.99, 0.6, 99)                   # ... but for 99 distinct above it
            sc[99:99 + tied[b]] = 0.55                             # and tied[b] rows at it
        if b == 7:
            sc[:] = 0.55                                          # every row ties
        rows = rng.choice(R, nk, replace=False)
        keep[b, :nk] = rows
        dets[b, 0, rows, -1] = rng.permutation(sc.astype(F32))
        nkeep[b] = nk
    out, guard, cnt = _launch_limit(dets, keep, nkeep, max_per_im, cap)
    check_limit(dets, keep, nkeep, max_per_im, cap, out, cnt)
    assert cnt.tolist()[:5] == [100, 101, 103, 105, 109] and cnt[5] == 60 and cnt[6] == 0 and cnt[7] == 250
    for b in range(B):
        assert (out[b, 0, min(int(cnt[b]), cap):] == SENTINEL).all(), b
    assert (guard == SENTINEL).all()
    perm = np.random.default_rng(4).permutation(B)
    out2, _, cnt2 = _launch_limit(np.ascontiguousarray(dets[perm]), np.ascontiguousarray(keep[perm]), nkeep[perm], max_per_im, cap)
    assert np.array_equal(cnt2, cnt[perm]) and np.array_equal(out2, out[perm])


# ------------------------------------------------------------------ training targets
class _RpnTrainCfg(object):
    RPN_STRADDLE_THRESH = 0
    RPN_POSITIVE_OVERLAP = 0.7
    RPN_NEGATIVE_OVERLAP = 0.3
    RPN_FG_FRACTION = 0.5
    RPN_BATCH_SIZE_PER_IM = 256


def _cmp_box_targets(got, ref, what):
    """dx / dy bit-exact; dw / dh (the log columns) to 8 ulp: numpy's fp32 log is ~4 ulp, CUDA's logf 1 ulp."""
    got, ref = got.reshape(-1, 4), ref.reshape(-1, 4)
    assert np.array_equal(got[:, :2], ref[:, :2]), what
    a, b = got[:, 2:], ref[:, 2:]
    assert (np.abs(a - b) <= 8 * np.spacing(np.maximum(np.abs(a), np.abs(b)).astype(F32))).all(), what


def check_rpn_targets(shapes, cells, strides, gt_boxes, gt_counts, im_info, tc, seed, out):
    for b in range(gt_boxes.shape[0]):
        lv = [(c, s, H, W) for c, s, (H, W) in zip(cells, strides, shapes)]
        g = gt_boxes[b, :gt_counts[b]] * F32(im_info[b, 2])
        ref, _ = ot.rpn_targets(lv, g, float(im_info[b, 0]), float(im_info[b, 1]), seed, b, straddle=float(tc.RPN_STRADDLE_THRESH),
                                pos=tc.RPN_POSITIVE_OVERLAP, neg=tc.RPN_NEGATIVE_OVERLAP, batch=int(tc.RPN_BATCH_SIZE_PER_IM),
                                fg_frac=tc.RPN_FG_FRACTION)
        for l, o in enumerate(out):
            assert np.array_equal(o['labels'][b].cpu().numpy(), ref[l]['labels']), (b, l)
            _cmp_box_targets(o['bbox_targets'][b].cpu().numpy(), ref[l]['bbox_targets'], 'image %d level %d' % (b, l))
            assert np.array_equal(o['inside'][b].cpu().numpy(), ref[l]['inside']), (b, l)
            assert np.array_equal(o['outside'][b].cpu().numpy(), ref[l]['outside']), (b, l)


def _synth_gt_tensors(B, seed, scale):
    import bench
    from detectandtrack_b200.modeling.trainer import pack_gt
    return pack_gt([dict(e, boxes=e['boxes'] / F32(scale)) for e in bench.synth_gt(B, 800, 1333, seed)])


@pytest.mark.parametrize('key', sorted(RPN_TARGETS, key=str), ids=lambda k: 'L%d-b%d' % (len(k[0]), k[3]))
def test_rpn_targets_full_size_vs_oracle(key):
    """dt_rpn_targets over the 5-level 800 x 1344 anchors (268 569 per image) of 2 clips with bench.synth_gt, one of them at
    a TRAIN.SCALES scale: labels, inside / outside weights bit-exact, box targets as _cmp_box_targets."""
    from detectandtrack_b200.ops import target_ops
    shapes, A, T, batch, fg, straddle = key
    cells = _cell_anchors(1)
    strides = [2. ** l for l in range(2, 7)]
    gt = _synth_gt_tensors(2, 11, 1.0)
    im_info = np.array([[800, 1333, 1.0], [800, 1333, 1.0]], F32)
    tc = _RpnTrainCfg()
    out = target_ops.rpn_targets(list(shapes), [torch.from_numpy(np.ascontiguousarray(c, F64)).cuda() for c in cells], strides, A,
                                 gt['rpn_boxes'], gt['rpn_counts'], torch.from_numpy(im_info).cuda(), tc, 9)
    check_rpn_targets(shapes, cells, strides, gt['rpn_boxes'].cpu().numpy(), gt['rpn_counts'].cpu().numpy(), im_info, tc, 9, out)


def check_sample_rois(rois, scores, counts, gt, im_info, cfg, seed, o):
    """oracle collect_train (the batch-wide top-N) then sample_rois per image on the device's own collect output."""
    from test_gpu_targets import _check_sampled
    tr = cfg.TRAIN
    B = rois.shape[0]
    kept = ot.collect_train([rois[b, :counts[b]] for b in range(B)], [scores[b, :counts[b]] for b in range(B)], int(tr.RPN_POST_NMS_TOP_N))
    g = {k: v.cpu().numpy() for k, v in gt.items()}
    for b in range(B):
        n = int(g['counts'][b])
        ref = ot.sample_rois(g['boxes'][b, :n], g['classes'][b, :n], g['crowd'][b, :n], g['keypoints'][b, :n], kept[b][:, 1:],
                             F32(im_info[b, 2]), b, seed, num_classes=int(cfg.MODEL.NUM_CLASSES), batch=int(tr.BATCH_SIZE_PER_IM),
                             fg_frac=tr.FG_FRACTION, fg_thresh=tr.FG_THRESH, bg_hi=tr.BG_THRESH_HI, bg_lo=tr.BG_THRESH_LO,
                             weights=tuple(cfg.MODEL.BBOX_REG_WEIGHTS), M=int(cfg.KRCNN.HEATMAP_SIZE))
        _check_sampled(o, b, ref, int(tr.BATCH_SIZE_PER_IM))


@pytest.mark.parametrize('key', sorted(SAMPLE), ids=lambda k: 'R%d-b%d' % (k[0], k[4]))
def test_sample_rois_on_device_collect_vs_oracle(key):
    """dt_sample_rois on the device's own training proposals: the 5-level RPN of 2 clips (K = 2000, grid logits), NMS and
    collect as the trainer runs them, then 512 RoIs per image and keypoint targets against oracle.targets.collect_train +
    sample_rois."""
    from detectandtrack_b200.ops import box_ops, rpn_ops, target_ops
    R, topn, T, K, batch, Gmax = key
    cfg = _train_cfg()
    cells = _cell_anchors(1)
    anchors = [torch.from_numpy(np.ascontiguousarray(c, F64)).cuda() for c in cells]
    outs = _rpn_inputs(1, A_FPN, FPN5, seed=21, pick=(0, 5))            # plain grid logits on both images
    im_info = np.array([[800, 1333, 1.0], [800, 1333, 1.0]], F32)
    props, counts = _launch_rpn(outs, anchors, im_info, topn, 0.0, 1, A_FPN, False)
    pd = torch.from_numpy(props).cuda()
    keep, nkeep = box_ops.nms_batched(pd.view(2 * 5, -1, 5), torch.from_numpy(counts).cuda().view(-1), 0.7, GE, BY_INDEX, max_keep=topn)
    rois, scores, rc = rpn_ops.collect(pd, keep, nkeep, topn)
    gt = _synth_gt_tensors(2, 13, 1.0)
    o = target_ops.sample_rois(rois, scores, rc, gt, torch.from_numpy(im_info).cuda(), cfg, 17, keypoints=True)
    check_sample_rois(rois.cpu().numpy(), scores.cpu().numpy(), rc.cpu().numpy(), gt, im_info, cfg, 17, o)


# ------------------------------------------------------------------ teacher-forced capture of the real steps
def _clone(r):
    """Outputs as the stage returned them (the step may later write into its buffers)."""
    if isinstance(r, torch.Tensor):
        return r.detach().clone()
    if isinstance(r, (list, tuple)):
        return type(r)(_clone(x) for x in r)
    if isinstance(r, dict):
        return {k: _clone(v) for k, v in r.items()}
    return r


def _capture(monkeypatch, mod, name, log):
    orig = getattr(mod, name)
    sig = inspect.signature(orig)

    def wrapped(*a, **kw):
        ba = sig.bind(*a, **kw)
        ba.apply_defaults()
        args = {k: (v.detach().clone() if isinstance(v, torch.Tensor) else v) for k, v in ba.arguments.items()}
        if name == 'sample_rois':
            args['gt'] = {k: v.clone() for k, v in args['gt'].items()}
        res = orig(*a, **kw)
        log.append((name, args, _clone(res)))
        return res
    monkeypatch.setattr(mod, name, wrapped)


def _np(t):
    return None if t is None else t.cpu().numpy()


def _check_captured(log, rec, tag):
    """Re-run the oracle on each captured stage's own inputs (bit-identical floats): keep lists, collect, levels, limit and
    targets equal; box decode inside its candidate bands."""
    done = {}
    band = 0
    for name, a, res in log:
        done[name] = done.get(name, 0) + 1
        if name == 'nms_batched':
            d = _np(a['dets'])
            check_nms(d, _np(a['counts']), a['thresh'], a['cmp_mode'], a['out_order'], a['max_keep'], _np(res[0]), _np(res[1]))
        elif name == 'collect':
            B, Lv, K, _ = a['props'].shape
            R = a['R'] or (a['post_nms_topn'] if a['post_nms_topn'] > 0 else Lv * K)
            check_collect(_np(a['props']), _np(a['keep']).reshape(B * Lv, K), _np(a['nkeep']).reshape(-1), a['post_nms_topn'], R,
                          _np(res[0]), _np(res[1]), _np(res[2]))
        elif name == 'distribute':
            r = _np(a['rois'])
            nd = len(r) if a['n_dev'] is None else int(_np(a['n_dev'])[0])
            check_distribute(r, nd, a['col0'], a['T'], a['k_min'], a['k_max'], a['s0'], a['lvl0'], _np(res[0]), _np(res[1]))
        elif name == 'box_decode':
            C = a['num_classes']
            band += check_box_decode(_np(a['rois']), _np(a['roi_counts']), _np(a['cls_logits']), _np(a['bbox_deltas']), C,
                                     _np(a['im_info']), _np(a['im_hw']), tuple(a['weights']), a['score_thresh'], a['T'],
                                     _np(res[0]), _np(res[1]))
        elif name == 'limit_detections':
            check_limit(_np(a['dets']), _np(a['keep']), _np(a['nkeep']), a['max_per_im'], a['cap'] or a['dets'].shape[2],
                        _np(res[0]), _np(res[1]))
        elif name == 'rpn_targets':
            check_rpn_targets(a['level_shapes'], [_np(c) for c in a['anchors']], a['strides'], _np(a['gt_boxes']), _np(a['gt_counts']),
                              _np(a['im_info']), a['cfg_train'], a['seed'], res)
        elif name == 'sample_rois':
            check_sample_rois(_np(a['rois']), _np(a['roi_scores']), _np(a['roi_counts']), a['gt'], _np(a['im_info']), a['cfg'],
                              a['seed'], res)
    rec('box_decode_rows_in_band_%s' % tag, band)
    print('%s: stages checked %s, box-decode rows inside the score band: %d' % (tag, sorted(done.items()), band))
    return done


def test_teacher_forced_real_steps(monkeypatch, record_property):
    """One r50fpn3d detect of 8 clips, one r18tube detect of 8 clips and one training step, with every box-stage call
    recorded; each downstream stage is then re-run by the oracle on the device's own upstream output and must agree."""
    import bench
    from detectandtrack_b200.modeling import params as Pm
    from detectandtrack_b200.modeling.engine import DetectionEngine
    from detectandtrack_b200.modeling.trainer import KeypointRcnnTrainer, pack_gt
    from detectandtrack_b200.ops import box_ops, rpn_ops, target_ops
    log = []
    for mod, names in ((rpn_ops, ('collect', 'distribute', 'box_decode', 'limit_detections')), (box_ops, ('nms_batched',)),
                       (target_ops, ('rpn_targets', 'sample_rois'))):
        for n in names:
            _capture(monkeypatch, mod, n, log)
    try:
        for wl in ('r50fpn3d', 'r18tube'):
            cfg = bench.bench_cfg(800, 1333, wl)
            blobs, spec = Pm.random_blobs(cfg)
            eng = DetectionEngine(cfg, blobs, spec, dtype='bf16')
            frames = torch.from_numpy(bench.synth_frames(8, bench.frames_per_clip(cfg), 800, 1333, 3)).cuda()
            del log[:]
            eng.detect_static(frames)
            torch.cuda.synchronize()
            done = _check_captured(log, record_property, wl)
            assert {'nms_batched', 'collect', 'box_decode', 'limit_detections'} <= set(done), done
            del eng
        cfg = _train_cfg()
        blobs, spec = Pm.random_blobs(cfg)
        tr = KeypointRcnnTrainer(cfg, blobs, spec)
        frames = torch.from_numpy(bench.synth_frames(2, 3, 800, 1333, 5)).cuda()
        del log[:]
        tr.step(frames, pack_gt(bench.synth_gt(2, 800, 1333, 11)), seed=9)
        torch.cuda.synchronize()
        done = _check_captured(log, record_property, 'train')
        assert {'rpn_targets', 'sample_rois', 'nms_batched', 'collect'} <= set(done), done
    finally:
        from test_gpu_engine import _cfg
        _cfg()
