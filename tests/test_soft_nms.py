"""CPU: TEST.SOFT_NMS / TEST.BBOX_VOTE without a GPU.
  * the oracle restatement (oracle/soft_nms.py) equals the reference's own soft_nms / box_voting, recorded in
    tests/golden/soft_nms.npz (tests/golden/gen_golden_soft_nms.py), bit for bit;
  * the np.average evaluation order the device kernel follows equals numpy's, so a numpy change shows up here;
  * dt_soft_nms_batched / dt_box_vote reject bad arguments on the host, before any CUDA call;
  * the engine and the test-time augmentation plan reject what the device box stage does not run, before anything
    is built."""
import os

import numpy as np
import pytest

from detectandtrack_b200 import _lib as L
from oracle import soft_nms as osn

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'soft_nms.npz')


def _cases(prefix):
    z = np.load(GOLDEN)
    return z, sorted({int(k.split('_')[0][1:]) for k in z.files if k.startswith(prefix)})


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def test_oracle_soft_nms_equals_reference_goldens():
    z, ks = _cases('s')
    methods = set()
    for k in ks:
        sigma, nt, th, m = z['s%d_params' % k]
        rows, inds = osn.soft_nms(z['s%d_dets' % k], sigma, nt, th, int(m))
        assert np.array_equal(_bits(rows), _bits(z['s%d_rows' % k])), k
        assert np.array_equal(inds, z['s%d_inds' % k]), k
        methods.add(int(m))
    assert methods == {0, 1, 2} and len(ks) >= 50


def test_oracle_box_voting_equals_reference_goldens():
    z, ks = _cases('v')
    for k in ks:
        got = osn.box_voting(z['v%d_top' % k], z['v%d_all' % k], z['v%d_thresh' % k])
        assert np.array_equal(_bits(got), _bits(z['v%d_voted' % k])), k


def test_soft_nms_tie_order_follows_the_discard_permutation():
    """Four equal scores, rows 0, 1 and 3 identical: row 1 decays to 0 and is replaced by row 3, which decays too and is
    replaced by row 2, so the survivors come out as [0, 2] -- the position order after discards, not the input order."""
    d = np.array([[0, 0, 9, 9, .9], [0, 0, 9, 9, .9], [20, 20, 29, 29, .9], [0, 0, 9, 9, .9]], np.float32)
    _, inds = osn.soft_nms(d, 0.5, 0.3, 0.001, 1)
    assert inds.tolist() == [0, 2]
    d[3] = [1, 1, 10, 10, .9]                      # overlaps row 0 by ~.68: decays, survives, lands after row 2
    _, inds = osn.soft_nms(d, 0.5, 0.3, 0.001, 1)
    assert inds.tolist() == [0, 2, 3]


def test_average_order_matches_numpy():
    rng = np.random.RandomState(0)
    sizes = list(range(1, 300)) + [511, 512, 513, 1000, 1024, 1025, 2047, 4096, 4099, 8191, 8192]
    for n in sizes:
        b = rng.uniform(0, 800, (n, 4)).astype(np.float32)
        w = rng.uniform(0.001, 1, n).astype(np.float32)
        assert np.array_equal(_bits(osn.weighted_average(b, w)), _bits(np.average(b, axis=0, weights=w))), n


def test_oracle_box_stage_options():
    """oracle/soft_nms.box_results_with_nms_and_limit: with both options off it is oracle/detections' stage; with
    soft-NMS and voting it is soft_nms -> box_voting -> the DETECTIONS_PER_IM limit, class by class."""
    from oracle import detections as odet
    rng = np.random.RandomState(3)
    n = 200
    x1, y1 = rng.uniform(0, 300, n), rng.uniform(0, 300, n)
    boxes = np.stack([x1, y1, x1 + rng.uniform(5, 80, n), y1 + rng.uniform(5, 80, n)], 1).astype(np.float32)
    boxes = np.concatenate([boxes, boxes], 1)
    p = rng.uniform(0, 1, n).astype(np.float32)
    scores = np.stack([1 - p, p], 1).astype(np.float32)
    a = odet.box_results_with_nms_and_limit(scores, boxes)
    b = osn.box_results_with_nms_and_limit(scores, boxes)
    assert np.array_equal(_bits(a[1]), _bits(b[1])) and np.array_equal(_bits(a[0]), _bits(b[0]))
    s = osn.box_results_with_nms_and_limit(scores, boxes, soft_nms=('linear', 0.5), bbox_vote=0.8)
    dets = np.hstack([boxes[p > 0.05, 4:], p[p > 0.05, None]]).astype(np.float32)
    rows = osn.box_voting(osn.soft_nms(dets, 0.5, 0.5, 0.0001, 1)[0], dets, 0.8)
    assert len(rows) > 100 and s[1].shape[0] == 100            # soft-NMS keeps more rows than the limit
    th = np.sort(rows[:, 4])[-100]
    assert np.array_equal(_bits(s[2][1]), _bits(rows[rows[:, 4] >= th]))


def _soft(**kw):
    a = dict(dets=None, batch=1, nmax=16, ld=5, counts=None, sigma=0.5, Nt=0.3, threshold=0.001, method=1, out=None,
             inds=None, counts_out=None, stream=None)
    a.update(kw)
    return L.lib().dt_soft_nms_batched(*a.values())


def _vote(**kw):
    a = dict(top=None, keep=None, top_counts=None, top_nmax=16, ld_top=5, all=None, all_counts=None, batch=1, nmax=16,
             ld=5, thresh=0.8, out=None, out_counts=None, stream=None)
    a.update(kw)
    return L.lib().dt_box_vote(*a.values())


P = 16        # a non-null (never dereferenced) pointer: every case below fails on the host first


@pytest.mark.parametrize('kw,msg', [
    (dict(method=3), b'method 3'),
    (dict(method=-1), b'method -1'),
    (dict(ld=4), b'ld >= 5'),
    (dict(nmax=8193), b'exceeds 8192'),
    (dict(nmax=-1), b'bad shape'),
    (dict(batch=-1), b'bad shape'),
    (dict(out=None, counts_out=P, dets=P), b'null output'),
    (dict(out=P, counts_out=None, dets=P), b'null output'),
    (dict(out=P, counts_out=P, dets=None), b'null dets'),
])
def test_soft_nms_rejects_bad_arguments_without_a_gpu(kw, msg):
    rc = _soft(**kw)
    err = L.lib().dt_last_error()
    assert rc != 0 and msg in err and b'dt_soft_nms_batched' in err, err


@pytest.mark.parametrize('kw,msg', [
    (dict(ld=4), b'ld, ld_top >= 5'),
    (dict(ld_top=3), b'ld, ld_top >= 5'),
    (dict(nmax=8193, top_nmax=8193), b'exceeds 8192'),
    (dict(top_nmax=-1), b'bad shape'),
    (dict(keep=P, top_nmax=8), b'must equal nmax'),
    (dict(top_counts=None, out=P, out_counts=P, all=P, top=P), b'null pointer'),
    (dict(top_counts=P, out=None, out_counts=P, all=P, top=P), b'null pointer'),
    (dict(top_counts=P, out=P, out_counts=P, all=None, top=P), b'null rows'),
    (dict(top_counts=P, out=P, out_counts=P, all=P, top=None), b'null rows'),
])
def test_box_vote_rejects_bad_arguments_without_a_gpu(kw, msg):
    rc = _vote(**kw)
    err = L.lib().dt_last_error()
    assert rc != 0 and msg in err and b'dt_box_vote' in err, err


def _engine_cfg(tube=False, **over):
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench
    cfg = bench.bench_cfg(96, 128, 'r18tube' if tube else 'r50fpn3d')
    for k, v in over.items():
        node = cfg
        parts = k.split('.')
        for p in parts[:-1]:
            node = node[p]
        node[parts[-1]] = v
    return cfg


@pytest.mark.parametrize('tube,over,exc,msg', [
    (False, {'TEST.SOFT_NMS.ENABLED': True, 'TEST.SOFT_NMS.METHOD': 'cosine'}, ValueError, 'Unknown soft_nms method: cosine'),
    (True, {'TEST.SOFT_NMS.ENABLED': True}, NotImplementedError, 'tube heads'),
    (True, {'TEST.BBOX_VOTE.ENABLED': True}, NotImplementedError, 'tube heads'),
])
def test_engine_rejects_before_anything_is_built(tube, over, exc, msg):
    from detectandtrack_b200.core.config import reset_cfg
    from detectandtrack_b200.modeling.engine import DetectionEngine
    try:
        cfg = _engine_cfg(tube, **over)
        with pytest.raises(exc, match=msg):
            DetectionEngine(cfg, blobs=None)       # no blobs, no device: the check runs first
    finally:
        reset_cfg()


def test_engine_check_accepts_what_it_runs():
    from detectandtrack_b200.core.config import reset_cfg
    from detectandtrack_b200.modeling import params as P_
    from detectandtrack_b200.modeling.engine import check_box_post
    try:
        for m in ('hard', 'linear', 'gaussian'):
            cfg = _engine_cfg(**{'TEST.SOFT_NMS.ENABLED': True, 'TEST.SOFT_NMS.METHOD': m, 'TEST.BBOX_VOTE.ENABLED': True})
            check_box_post(cfg, P_.GraphSpec(cfg))
        cfg = _engine_cfg(tube=True, **{'TEST.SOFT_NMS.METHOD': 'cosine'})        # disabled options are not read
        check_box_post(cfg, P_.GraphSpec(cfg))
    finally:
        reset_cfg()


def test_view_plan_rejects_unknown_method():
    from detectandtrack_b200.core import tta
    from detectandtrack_b200.core.config import reset_cfg
    try:
        cfg = _engine_cfg(**{'TEST.COMPETITION_MODE': True, 'TEST.BBOX_AUG.SCORE_HEUR': 'UNION',
                             'TEST.BBOX_AUG.COORD_HEUR': 'UNION', 'TEST.SOFT_NMS.ENABLED': True,
                             'TEST.SOFT_NMS.METHOD': 'Linear'})
        with pytest.raises(ValueError, match='Unknown soft_nms method: Linear'):
            tta.view_plan(cfg, None, 96, 128)
    finally:
        reset_cfg()
