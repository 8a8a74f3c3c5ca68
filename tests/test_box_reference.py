"""CPU: the host references the box-stage value tests (tests/test_gpu_box_step.py) compare csrc/proposals.cu, csrc/boxes.cu
and csrc/targets.cu with, where oracle/ does not already provide one: the RPN top-k under the documented tie rule (the
time-major tube score included), the 2-D decode and the softmax score as the sets of fp32 values the kernels may produce, and
the DETECTIONS_PER_IM limit with the detection-slot cap.  Each is pinned here once against the oracle (itself pinned to the
reference's goldens by tests/test_oracle_*.py) or the goldens.

Exactness by construction (the RPN score).  The kernel scores an anchor as 1 / (1 + expf(-x)) in fp32; expf is within 2 ulp
of exp, so the host cannot reproduce the score's last bit, but it does not need to for the ranking.  The tests draw logits on
a coarse grid, multiples of 1/8 in [-8, 8], plus saturated values >= 17:
  * two distinct grid logits are >= 1/8 apart, and a time-major mean of T = 3 grid logits (an exact fp32 sum of multiples of
    1/8, then / 3) moves by >= 1/24 between distinct sums.  sigmoid' >= sigmoid'(8) = 3.35e-4 on [-8, 8], so the fp64
    sigmoids of distinct keys are >= 3.35e-4 / 24 = 1.4e-5 apart, while the device score is within 4 u = 2.4e-7 of it
    (expf's 2 ulp carried through 1 + e, one rounding there and one in the division): distinct keys keep their order;
  * equal keys give bit-equal device scores (the same fp32 operations on the same fp32 inputs);
  * for x >= 17, expf(-x) <= 4.2e-8 < 2^-24, so 1 + expf(-x) rounds to 1 and the score is exactly 1.0: every such anchor
    ties, above every grid key (sigmoid(8) < 1 - 2^-12).
So the device ranking equals the host's (key descending, anchor index ascending) exactly.  Means in (8, 17) would break the
argument (their sigmoids crowd within an ulp of 1) and are rejected by rank_keys.

NaN logits are outside these tests: the kernel's sort key maps a NaN score above +inf, so a NaN anchor from a diverged run
is selected first, where numpy's argsort(-s) would put it last."""
import os

import numpy as np
import pytest

from oracle import boxes as obox
from oracle import detections as odet
from oracle import proposals as oprop

F32, F64 = np.float32, np.float64
GOLDEN = os.path.join(os.path.dirname(__file__), 'golden')
SAT = 17.0                       # logits (means) at or above this saturate to a score of exactly 1.0
EXP_STEPS = 3                    # expf's 2 ulp plus the host reference's 0.5 ulp, in whole fp32 steps (see exp_candidates)


# ------------------------------------------------------------------ RPN ranking
def grid_logits(rng, shape):
    """Multiples of 1/8 in [-8, 8] (exact in fp32 and bf16)."""
    return (rng.integers(-64, 65, shape) / 8.0).astype(F32)


def time_mean(logits_t):
    """[T, n] fp32 -> the kernel's tube score argument: sequential fp32 sum over T, then / T in fp32."""
    acc = np.asarray(logits_t[0], F32).copy()
    for t in range(1, len(logits_t)):
        acc = (acc + np.asarray(logits_t[t], F32)).astype(F32)
    return (acc / F32(len(logits_t))).astype(F32)


def rank_keys(x):
    """Ranking keys of fp32 sigmoid arguments (module docstring): the argument itself on [-8, 8], +inf (one tie class) at or
    above SAT.  Anything else has no exact ranking on the device and is refused."""
    x = np.asarray(x, F64)
    ok = (np.abs(x) <= 8.0) | (x >= SAT)
    assert ok.all(), 'sigmoid argument outside [-8, 8] and below %g: %s' % (SAT, x[~ok][:4])
    return np.where(x >= SAT, np.inf, x)


def topk_ref(keys, K):
    """Anchor indices of the top K: descending key, then ascending index (the kernel's documented tie rule)."""
    keys = np.asarray(keys, F64)
    order = np.lexsort((np.arange(len(keys)), -keys))
    return order[:min(K, len(keys)) if K > 0 else len(keys)]


def sigmoid_tol(x):
    """|device score - fp64 sigmoid|: expf's 2 ulp relative error e moves 1 + e by <= 2^-22 e <= 2^-22; the add and the
    division round once each (2^-24 relative each); the result is <= 1: 4 * 2^-24 absolute, times sigmoid for small x."""
    return 4 * 2.0 ** -24 * np.maximum(1.0 / (1.0 + np.exp(-np.asarray(x, F64))), 2.0 ** -126)


# ------------------------------------------------------------------ fp32 exp as a set of candidates
def exp_candidates(x):
    """[2*EXP_STEPS + 1, ...] fp32: the values a <= 2 ulp expf(x) can take.  fp32(exp(x)) in fp64 is within 0.5 ulp of e^x;
    expf is within 2 ulp of e^x, so within 2.5 ulp of fp32(exp(x)); both are fp32 values, and where an ulp boundary (a
    power of two) lies between them the steps below it are half as wide, so 3 nextafter steps either way cover it."""
    e = np.exp(np.asarray(x, F64)).astype(F32)
    out = [e]
    up, dn = e.copy(), e.copy()
    for _ in range(EXP_STEPS):
        up = np.nextafter(up, F32(np.inf)); dn = np.nextafter(dn, F32(0))
        out = [dn.copy()] + out + [up.copy()]
    return np.stack(out)


def decode2d(boxes, deltas, weights, clip, exp_fn):
    """lib/utils/boxes.py:141-183 in fp32, operation by operation as decode_f32 of csrc/proposals.cu evaluates it, with
    exp supplied: boxes [n, 4] fp32, deltas [n, 4] fp32 -> [n, 4] fp32 (before clipping)."""
    b, d = np.asarray(boxes, F32), np.asarray(deltas, F32)
    wx, wy, ww, wh = [F32(w) for w in weights]
    w = (b[:, 2] - b[:, 0]) + F32(1); h = (b[:, 3] - b[:, 1]) + F32(1)
    cx = b[:, 0] + F32(0.5) * w; cy = b[:, 1] + F32(0.5) * h
    dx, dy = d[:, 0] / wx, d[:, 1] / wy
    dw, dh = np.minimum(d[:, 2] / ww, F32(clip)), np.minimum(d[:, 3] / wh, F32(clip))
    pcx, pcy = dx * w + cx, dy * h + cy
    pw, ph = exp_fn(dw) * w, exp_fn(dh) * h
    return np.stack([pcx - F32(0.5) * pw, pcy - F32(0.5) * ph, pcx + F32(0.5) * pw, pcy + F32(0.5) * ph], -1).astype(F32)


def decode2d_set(boxes, deltas, weights, clip):
    """[7, n, 4]: the 2-D decode with every exp candidate.  x1 / x2 depend on exp(dw) alone and y1 / y2 on exp(dh) alone,
    so candidate k of a coordinate is the decode with the k-th exp value, and the device coordinate must be one of the 7.
    This is the per-coordinate error band of the fp32 decode: the only non-correctly-rounded step is expf, and the band is
    the image of its 2 ulp through the following fp32 multiply, halving, add / subtract and clip."""
    ex = exp_candidates
    return np.stack([decode2d(boxes, deltas, weights, clip, lambda v, k=k: ex(v)[k]) for k in range(2 * EXP_STEPS + 1)])


def clip_boxes(b, h, w):
    """clip_tiled_boxes (boxes.py:243-253) on [..., 4T] fp32; h, w are the image's fp32 height and width."""
    b = np.array(b, F32, copy=True)
    h1, w1 = F32(F32(h) - F32(1)), F32(F32(w) - F32(1))
    b[..., 0::4] = np.maximum(np.minimum(b[..., 0::4], w1), F32(0)); b[..., 2::4] = np.maximum(np.minimum(b[..., 2::4], w1), F32(0))
    b[..., 1::4] = np.maximum(np.minimum(b[..., 1::4], h1), F32(0)); b[..., 3::4] = np.maximum(np.minimum(b[..., 3::4], h1), F32(0))
    return b


def filter_ok(b, min_size, im_info):
    """_filter_boxes (generate_proposals.py:184-196) per row of [..., 4T] fp32, AND over the frames."""
    ok = None
    for t in range(b.shape[-1] // 4):
        f = b[..., 4 * t:4 * t + 4].reshape(-1, 4)
        o = np.zeros(len(f), bool)
        o[oprop.filter_boxes(f, min_size, im_info)] = True
        o = o.reshape(b.shape[:-1])
        ok = o if ok is None else ok & o
    return ok


def rpn_ref(keys, deltas, anchors, im_info, K, min_size, T):
    """generate_proposals.py:40-114 up to NMS for one image and level.  keys [n] (rank_keys), deltas [n, 4T] fp32 and
    anchors [n, 4T] fp64 in anchor order (H, W, A).  Returns dict(idx [K'] selected anchors in output order, boxes
    [S, K', 4T] candidate boxes (S = 7 for 2-D, 1 for the fp64 tube decode, which rounds once and is exact), state [K']:
    1 kept, 0 filtered, -1 kept for some candidates and not others)."""
    im_info = np.asarray(im_info, F32)
    idx = topk_ref(keys, K)
    d, a = np.asarray(deltas, F32)[idx], np.asarray(anchors, F64)[idx]
    if T == 1:
        cand = decode2d_set(a.astype(F32), d, (1., 1., 1., 1.), obox.BBOX_XFORM_CLIP)
    else:
        cand = obox.bbox_transform(a, d, (1., 1., 1., 1.))[None]
    cand = clip_boxes(cand, im_info[0], im_info[1])
    ok = np.stack([filter_ok(c, min_size, im_info) for c in cand])
    state = np.where(ok.all(0), 1, np.where(ok.any(0), -1, 0))
    return dict(idx=idx, boxes=cand, state=state)


def match_rows(rows, ref, scores):
    """Walk the reference candidates in order against the device rows [m, 4T+1] (the count's worth): a kept candidate is the
    next row, a filtered one is absent, an undecided one (state -1) is the next row if that row is one of its candidate
    boxes.  Every matched row's box must be a candidate coordinate by coordinate and its score must equal `scores[j]`
    bit for bit.  Returns the number of undecided candidates."""
    r, und = 0, 0
    for j in range(len(ref['idx'])):
        st = ref['state'][j]
        hit = r < len(rows) and bool((rows[r, :-1][None] == ref['boxes'][:, j]).any(0).all())
        if st == -1:
            und += 1
        if st == 1 or (st == -1 and hit):
            assert hit, ('row %d: box %s not among the candidates of anchor %d' % (r, rows[r, :-1] if r < len(rows) else None,
                                                                                     ref['idx'][j]))
            assert rows[r, -1] == scores[j], (r, rows[r, -1], scores[j])
            r += 1
    assert r == len(rows), ('extra device rows', r, len(rows))
    return und


# ------------------------------------------------------------------ box head score
def softmax_candidates(logits, j):
    """[7, n] fp32: the values box_decode_kernel's softmax score of class j can take for logits [n, C] fp32 (C = 2, the
    model's): m = max, e_c = expf(l_c - m) (the difference rounds in fp32 here as on the device; e = 1 exactly for the
    maximum), sum = (0 + e_0)
    + e_1, score = e_j / sum, all fp32.  The one inexact step is expf of the non-maximal class, so the score band is that
    exp's candidate set carried through the add and the division."""
    l = np.asarray(logits, F32)
    assert l.shape[1] == 2
    m = l.max(1)
    d = (l - m[:, None]).astype(F32)
    out = []
    for k in range(2 * EXP_STEPS + 1):
        e = np.where(d == 0, F32(1), exp_candidates(d)[k]).astype(F32)
        s = (F32(0) + e[:, 0]).astype(F32) + e[:, 1]
        out.append((e[:, j] / s).astype(F32))
    return np.stack(out)


def score_filter_state(cand, thresh):
    """Per row: 1 kept by 'score > thresh' for every candidate, 0 for none, -1 inside the band (decided by the device's own
    score, which must then be self-consistent)."""
    gt = cand > F32(thresh)
    return np.where(gt.all(0), 1, np.where(gt.any(0), -1, 0))


# ------------------------------------------------------------------ DETECTIONS_PER_IM limit with the cap
def limit_ref(class_scores, max_per_im, cap):
    """lib/core/test.py:790-800 on one image's per-class score lists (each in NMS keep order): if more than max_per_im rows
    survive, keep those with score >= the max_per_im-th largest (every row tied at it).  Returns per class (count, kept
    positions in keep order): the count is the full kept count, the positions the first `cap` of them (the rows
    dt_limit_detections writes)."""
    allsc = np.concatenate([np.asarray(s, F32) for s in class_scores]) if class_scores else np.zeros(0, F32)
    th = -np.inf
    if max_per_im > 0 and len(allsc) > max_per_im:
        th = np.sort(allsc)[-max_per_im]
    out = []
    for s in class_scores:
        pos = np.where(np.asarray(s, F32) >= th)[0]
        out.append((len(pos), pos[:cap]))
    return out


# ================================================================== pins
def _gp(tag):
    return dict(np.load(os.path.join(GOLDEN, tag + '.npz')))


@pytest.mark.parametrize('tag', ['gp2d', 'gp3d'])
def test_rpn_ref_matches_oracle_generate_proposals(tag):
    """rpn_ref on the goldens' RPN outputs equals oracle.generate_proposals before NMS: the same anchors in the same order
    (distinct scores: the tie rule is not exercised), every 2-D box among its candidates (the oracle's own exp is numpy's
    fp32 exp), tube boxes bit-exact, and the same rows filtered."""
    g = _gp(tag)
    sc, dl, im = g[tag + '_scores'][0], g[tag + '_deltas'][0], g[tag + '_im_info'][0]
    stride = float(g[tag + '_stride'])
    ga = _gp('anchors')
    cell = ga['anchors_fpn5'] if tag == 'gp2d' else ga['anchors_rpn12_T3']
    T = cell.shape[1] // 4
    H, W = sc.shape[-2:]
    keys = sc.transpose(1, 2, 0).reshape(-1).astype(F64)
    deltas = dl.transpose(1, 2, 0).reshape(-1, 4 * T)
    anchors = oprop.shifted_anchors(cell, H, W, stride, T)
    for K, min_size in ((1000, 0.0), (300, 16.0), (-1, 0.0)):
        ref = rpn_ref(keys, deltas, anchors, im, K, min_size, T)
        _, _, (pre_p, pre_s), _ = oprop.generate_proposals(sc, dl, im, cell, stride, K, 0, 0.7, min_size, return_intermediate=True)
        kept = ref['state'] != 0
        assert (ref['state'] != -1).all()
        assert kept.sum() == len(pre_p)
        got = ref['boxes'][:, kept]
        assert ((got == pre_p[None]).any(0)).all()
        if T > 1:
            assert np.array_equal(got[0], pre_p)
        assert np.array_equal(keys[ref['idx'][kept]].astype(F32), pre_s[:, 0])


def test_topk_tie_rule_and_time_mean():
    """Ties: descending key, ascending index; saturated keys tie above every grid key; the tube mean is the sequential fp32
    sum / T (not numpy's pairwise mean, which differs in the last bit for some triples)."""
    keys = rank_keys(np.array([1.0, 17.0, 1.0, 30.0, -8.0, 8.0, 1.0, 17.5], F32))
    assert topk_ref(keys, 5).tolist() == [1, 3, 7, 5, 0]
    assert topk_ref(keys, -1).tolist() == [1, 3, 7, 5, 0, 2, 6, 4]
    with pytest.raises(AssertionError):
        rank_keys(np.array([9.0], F32))
    lt = np.array([[0.1, 17.0], [0.2, 20.0], [0.3, 30.0]], F32)
    m = time_mean(lt)
    assert m[0] == F32(F32(F32(F32(0.1) + F32(0.2)) + F32(0.3)) / F32(3))
    # grid means: distinct sums stay distinct and ordered after the fp32 division
    rng = np.random.default_rng(0)
    g = grid_logits(rng, (3, 20000))
    s = (g[0].astype(F64) + g[1] + g[2])
    mm = time_mean(g).astype(F64)
    o = np.argsort(s, kind='stable')
    assert (np.diff(mm[o]) >= 0).all() and ((np.diff(s[o]) > 0) == (np.diff(mm[o]) > 0)).all()


def test_sigmoid_separation_argument():
    """The numbers of the module docstring: grid neighbours (and tube means 1/24 apart) are separated by more than twice the
    device score's error, and a saturated anchor's expf(-17) is below half an ulp of 1 even at 2 ulp error."""
    x = np.arange(-8 * 24, 8 * 24 + 1) / 24.0
    s = 1.0 / (1.0 + np.exp(-x))
    assert (np.diff(s) > 2 * (sigmoid_tol(x[:-1]) + sigmoid_tol(x[1:]))).all()
    assert np.exp(-17.0) * (1 + 2.0 ** -22) < 2.0 ** -24
    assert F32(1) / (F32(1) + F32(np.exp(-17.0))) == F32(1)
    assert 1.0 / (1.0 + np.exp(-8.0)) < 1 - 2.0 ** -12


def test_decode2d_set_contains_oracle_decode():
    """The candidate set contains the oracle's fp32 bbox_transform (numpy's own fp32 exp) on the goldens' RoIs and random
    deltas, including deltas past BBOX_XFORM_CLIP, and candidate 3 is the correctly rounded exp."""
    g = dict(np.load(os.path.join(GOLDEN, 'cd2d.npz')))
    rng = np.random.default_rng(1)
    boxes = g['cd2d_rois'][:, 1:].astype(F32)
    d = rng.normal(0, 1.5, boxes.shape).astype(F32)
    d[::7, 2:] = 9.0                                            # past the clip
    for wts in ((1., 1., 1., 1.), (10., 10., 5., 5.)):
        cand = decode2d_set(boxes, d, wts, obox.BBOX_XFORM_CLIP)
        ref = obox.bbox_transform(boxes, d, wts)
        assert (cand == ref[None]).any(0).all()
        exact = decode2d(boxes, d, wts, obox.BBOX_XFORM_CLIP, lambda v: np.exp(v.astype(F64)).astype(F32))
        assert np.array_equal(cand[EXP_STEPS], exact)
    e = exp_candidates(np.array([0.0, 1.0, np.log(2.0)], F32))
    assert e.shape == (7, 3) and (np.diff(e, axis=0) > 0).all()


def test_softmax_candidates_contain_oracle_softmax():
    rng = np.random.default_rng(2)
    l = rng.normal(0, 3, (5000, 2)).astype(F32)
    l[:10, 1] = l[:10, 0]                                       # a tie: both 0.5
    cand = softmax_candidates(l, 1)
    p = odet.softmax(l)[:, 1]
    # the oracle's softmax (numpy's fp32 exp, the same fp32 differences and sum) lies inside the band's hull
    assert ((p >= cand.min(0)) & (p <= cand.max(0))).all()
    assert (cand[:, :10] == F32(0.5)).all()
    st = score_filter_state(cand, 0.05)
    assert set(np.unique(st)) <= {-1, 0, 1}


@pytest.mark.parametrize('ties', [0, 1, 3, 5])
def test_limit_ref_matches_oracle(ties):
    """limit_ref's counts equal oracle.detections.box_results_with_nms_and_limit's per-class rows (one class, no NMS:
    distinct boxes far apart), with `ties` extra rows tied at the threshold, and the write cut at cap."""
    rng = np.random.default_rng(3 + ties)
    n = 130
    sc = rng.permutation(np.linspace(0.06, 0.99, n)).astype(F32)
    srt = np.sort(sc)
    th = srt[-100]
    sc[np.where(sc < th)[0][:ties]] = th                       # more rows at the 100th score
    boxes = np.zeros((n, 8), F32)
    boxes[:, 4] = np.arange(n) * 50; boxes[:, 5] = 0; boxes[:, 6] = np.arange(n) * 50 + 10; boxes[:, 7] = 10
    scores = np.zeros((n, 2), F32); scores[:, 1] = sc
    _, _, cls = odet.box_results_with_nms_and_limit(scores, boxes, 2, 0.05, 0.5, 100)
    order = np.array(obox.nms(np.hstack((boxes[:, 4:], sc[:, None])), 0.5))
    (cnt, pos), = limit_ref([sc[order]], 100, 104)
    assert cnt == len(cls[1]) == 100 + ties
    assert np.array_equal(sc[order][pos], cls[1][:104, -1])
    (cnt2, pos2), = limit_ref([sc[order]], 100, 102)
    assert cnt2 == cnt and len(pos2) == min(cnt, 102)


def test_nms_and_collect_distribute_oracle_pins():
    """The oracle pieces the GPU file uses directly, pinned once more at the goldens: nms on nms2d / nmst3, collect and
    distribute on cd2d / cd3d (levels and restore index)."""
    n = dict(np.load(os.path.join(GOLDEN, 'nms2d.npz')))
    for th in (3, 5, 7):
        assert np.array_equal(obox.nms(n['nms2d_dets'], th / 10.), n['nms2d_keep_%d' % th])
    t = dict(np.load(os.path.join(GOLDEN, 'nmst3.npz')))
    for th in (3, 5, 7):
        assert np.array_equal(np.sort(obox.nms(t['nmst3_dets'], th / 10.)), np.sort(t['nmst3_keep_%d' % th]))
    for tag in ('cd2d', 'cd3d'):
        g = dict(np.load(os.path.join(GOLDEN, tag + '.npz')))
        rois = oprop.collect([g['%s_in_rois%d' % (tag, i)] for i in range(5)], [g['%s_in_scores%d' % (tag, i)] for i in range(5)], 1000)
        assert np.array_equal(rois, g[tag + '_rois'])
        lv = oprop.map_rois_to_fpn_levels(rois[:, 1:])
        assert np.array_equal(lv, g[tag + '_lvls'])
        _, _, restore = oprop.distribute(rois)
        assert np.array_equal(restore, g[tag + '_idx_restore'])
