"""GPU: dt_soft_nms_batched and dt_box_vote (TEST.SOFT_NMS / TEST.BBOX_VOTE) bit for bit against oracle/soft_nms.py
(itself pinned to the reference by tests/test_soft_nms.py) and, where oracle/_ref is built, the compiled reference live:
at the benchmarked step's shape (8 lists x 1000 rows), at DT_NMS_MAX_BOXES rows, on the golden edge sets, through the
drop-in host surface, teacher-forced on the captured configs[3]-shaped step (plain and with a 2-view H_FLIP plan), and on
the whole path of the small clip.  With both options off the step launches no new kernel."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import soft_nms as osn

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'soft_nms.npz')
METHODS = ('hard', 'linear', 'gaussian')


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _realistic(rng, n, w=1333, h=800):
    """Box-head-like rows: many proposals around a few objects, scores over SCORE_THRESH."""
    if n == 0:
        return np.zeros((0, 5), np.float32)
    k = rng.randint(0, max(1, n // 40), n)
    cx, cy = rng.uniform(0, w, k.max() + 1)[k], rng.uniform(0, h, k.max() + 1)[k]
    bw, bh = rng.uniform(20, 300, k.max() + 1)[k], rng.uniform(40, 400, k.max() + 1)[k]
    x1 = np.clip(cx - bw / 2 + rng.normal(0, 8, n), 0, w - 1); y1 = np.clip(cy - bh / 2 + rng.normal(0, 8, n), 0, h - 1)
    x2 = np.clip(x1 + bw * rng.uniform(.8, 1.2, n), 0, w - 1); y2 = np.clip(y1 + bh * rng.uniform(.8, 1.2, n), 0, h - 1)
    return np.stack([x1, y1, x2, y2, rng.uniform(0.05, 1, n)], 1).astype(np.float32)


def _ref_module():
    try:
        from oracle._ref import cython_nms
        return cython_nms
    except ImportError:
        return None


def _device_soft(lists, nmax, sigma, nt, th, method):
    from detectandtrack_b200.ops import box_ops
    B = len(lists)
    d = np.zeros((B, nmax, 5), np.float32)
    for b, x in enumerate(lists):
        d[b, :len(x)] = x
    cnt = torch.tensor([len(x) for x in lists], dtype=torch.int32, device='cuda')
    rows, inds, num = box_ops.soft_nms_batched(torch.from_numpy(d).cuda(), cnt, sigma, nt, th, method)
    torch.cuda.synchronize()
    return rows.cpu().numpy(), inds.cpu().numpy(), num.cpu().numpy(), d, cnt


def _check_soft(lists, nmax, sigma, nt, th, method, live=True):
    rows, inds, num, d, cnt = _device_soft(lists, nmax, sigma, nt, th, method)
    cn = _ref_module() if live else None
    for b, x in enumerate(lists):
        r, i = osn.soft_nms(x, sigma, nt, th, osn.METHODS[method])
        n = int(num[b])
        assert n == len(r), (b, method, n, len(r))
        assert np.array_equal(_bits(rows[b, :n]), _bits(r)), (b, method)
        assert np.array_equal(inds[b, :n], i), (b, method)
        if cn is not None and len(x):
            rr, ri = cn.soft_nms(np.ascontiguousarray(x), np.float32(sigma), np.float32(nt), np.float32(th),
                                 np.uint8(osn.METHODS[method]))
            assert np.array_equal(_bits(rows[b, :n]), _bits(rr)) and np.array_equal(inds[b, :n], ri), (b, method, 'live')
    return rows, inds, num, d, cnt


@pytest.mark.parametrize('method', METHODS)
def test_soft_nms_step_shape_exact(method):
    """configs[3]: 8 images x 1000 rows of one foreground class; ragged counts, one empty list."""
    rng = np.random.RandomState(11)
    lists = [_realistic(rng, n) for n in (1000, 1000, 999, 640, 1000, 1, 0, 1000)]
    _check_soft(lists, 1000, 0.5, 0.5, 0.0001, method)


@pytest.mark.parametrize('method', ['linear', 'gaussian'])
def test_soft_nms_max_boxes_exact(method):
    """DT_NMS_MAX_BOXES rows in one list (a test-time augmentation union can be this long)."""
    rng = np.random.RandomState(12)
    _check_soft([_realistic(rng, 8192)], 8192, 0.5, 0.3, 0.0001, method, live=False)


def test_soft_nms_golden_edge_sets():
    z = np.load(GOLDEN)
    for k in sorted({int(x.split('_')[0][1:]) for x in z.files if x.startswith('s')}):
        sigma, nt, th, m = z['s%d_params' % k]
        d = z['s%d_dets' % k]
        rows, inds, num, _, _ = _device_soft([d], max(len(d), 1), sigma, nt, th, METHODS[int(m)])
        n = int(num[0])
        assert np.array_equal(_bits(rows[0, :n]), _bits(z['s%d_rows' % k])), k
        assert np.array_equal(inds[0, :n], z['s%d_inds' % k]), k


def _vote_ref(top, alld, th):
    return osn.box_voting(top, alld, th)


def test_box_vote_after_hard_nms_step_shape_exact():
    from detectandtrack_b200.ops import box_ops
    rng = np.random.RandomState(13)
    lists = [_realistic(rng, n) for n in (1000, 1000, 700, 1000, 3, 1000, 0, 1000)]
    d = np.zeros((8, 1000, 5), np.float32)
    for b, x in enumerate(lists):
        d[b, :len(x)] = x
    dt = torch.from_numpy(d).cuda()
    cnt = torch.tensor([len(x) for x in lists], dtype=torch.int32, device='cuda')
    keep, nkeep = box_ops.nms_batched(dt, cnt, 0.5, box_ops.NMS_2D_GE, box_ops.ORDER_INDEX)
    for th in (0.8, 0.5):
        rows, num = box_ops.box_vote(dt, cnt, th, keep=keep, nkeep=nkeep)
        rows, num, kp, nk = rows.cpu().numpy(), num.cpu().numpy(), keep.cpu().numpy(), nkeep.cpu().numpy()
        for b, x in enumerate(lists):
            assert num[b] == nk[b]
            top = x[kp[b, :nk[b]]]
            assert np.array_equal(_bits(rows[b, :num[b]]), _bits(_vote_ref(top, x, th))), (b, th)


@pytest.mark.parametrize('n', [1000, 8192])
def test_box_vote_after_soft_nms_exact(n):
    from detectandtrack_b200.ops import box_ops
    rng = np.random.RandomState(14)
    B = 8 if n == 1000 else 1
    lists = [_realistic(rng, n) for _ in range(B)]
    rows, _, num, d, cnt = _device_soft(lists, n, 0.5, 0.5, 0.0001, 'linear')
    dt = torch.from_numpy(d).cuda()
    top = torch.from_numpy(rows).cuda()
    voted, vnum = box_ops.box_vote(dt, cnt, 0.8, top=top, top_counts=torch.from_numpy(num).cuda())
    voted, vnum = voted.cpu().numpy(), vnum.cpu().numpy()
    for b, x in enumerate(lists):
        assert vnum[b] == num[b]
        assert np.array_equal(_bits(voted[b, :num[b]]), _bits(_vote_ref(rows[b, :num[b]], x, 0.8))), b


def test_box_vote_golden_sets_and_host_surface():
    from detectandtrack_b200.utils import boxes as ub
    z = np.load(GOLDEN)
    for k in sorted({int(x.split('_')[0][1:]) for x in z.files if x.startswith('v')}):
        got = ub.box_voting(z['v%d_top' % k], z['v%d_all' % k], z['v%d_thresh' % k])
        assert np.array_equal(_bits(got), _bits(z['v%d_voted' % k])), k


def test_nms_wrapper_soft_nms_matches_reference_surface():
    from detectandtrack_b200.core import nms_wrapper as nw
    rng = np.random.RandomState(15)
    d = _realistic(rng, 300)
    cn = _ref_module()
    for m in METHODS:
        rows, inds = nw.soft_nms(d, sigma=0.5, overlap_thresh=0.3, score_thresh=0.001, method=m)
        r, i = osn.soft_nms(d, 0.5, 0.3, 0.001, osn.METHODS[m])
        assert rows.dtype == np.float32 and inds.dtype == np.int64
        assert np.array_equal(_bits(rows), _bits(r)) and np.array_equal(inds, i), m
        if cn is not None:
            rr, ri = cn.soft_nms(d, np.float32(0.5), np.float32(0.3), np.float32(0.001), np.uint8(osn.METHODS[m]))
            assert np.array_equal(_bits(rows), _bits(rr)) and np.array_equal(inds, ri), m
    empty = np.zeros((0, 5), np.float32)
    assert nw.soft_nms(empty) is empty
    with pytest.raises(NotImplementedError, match='tubes'):
        nw.soft_nms(np.zeros((3, 13), np.float32))
    with pytest.raises(AssertionError, match='Unknown soft_nms method'):
        nw.soft_nms(d, method='cosine')


# ------------------------------------------------------------------ the captured step
SETTINGS = {'off': {}, 'soft_linear': {'TEST.SOFT_NMS.ENABLED': True, 'TEST.SOFT_NMS.METHOD': 'linear'},
            'soft_gaussian': {'TEST.SOFT_NMS.ENABLED': True, 'TEST.SOFT_NMS.METHOD': 'gaussian'},
            'soft_hard': {'TEST.SOFT_NMS.ENABLED': True, 'TEST.SOFT_NMS.METHOD': 'hard'},
            'vote': {'TEST.BBOX_VOTE.ENABLED': True},
            'soft_vote': {'TEST.SOFT_NMS.ENABLED': True, 'TEST.SOFT_NMS.METHOD': 'linear', 'TEST.BBOX_VOTE.ENABLED': True}}


def _set(cfg, over):
    for k, v in over.items():
        node = cfg
        parts = k.split('.')
        for p in parts[:-1]:
            node = node[p]
        node[parts[-1]] = v


def _oracle_post(cfg, dets, cnt):
    """oracle/soft_nms.box_results_with_nms_and_limit on the step's own decoded rows of one image (one foreground
    class): every row is already over SCORE_THRESH, so the threshold is disabled."""
    rows = dets[:cnt]
    scores = np.stack([1 - rows[:, 4], rows[:, 4]], 1).astype(np.float32)
    boxes = np.concatenate([rows[:, :4], rows[:, :4]], 1)
    soft = (cfg.TEST.SOFT_NMS.METHOD, cfg.TEST.SOFT_NMS.SIGMA) if cfg.TEST.SOFT_NMS.ENABLED else None
    vote = cfg.TEST.BBOX_VOTE.VOTE_TH if cfg.TEST.BBOX_VOTE.ENABLED else None
    _, _, cls_boxes = osn.box_results_with_nms_and_limit(scores, boxes, 2, -np.inf, cfg.TEST.NMS,
                                                         cfg.TEST.DETECTIONS_PER_IM, soft_nms=soft, bbox_vote=vote)
    return cls_boxes[1]


@pytest.mark.parametrize('plan_flip', [False, True], ids=['plain', 'hflip_union'])
def test_captured_step_teacher_forced(plan_flip):
    sys.path.insert(0, ROOT)
    import bench
    from detectandtrack_b200.core import tta
    from detectandtrack_b200.core.config import reset_cfg
    from detectandtrack_b200.modeling import params as Pm
    from detectandtrack_b200.modeling.engine import DetectionEngine
    B, H, W = (8, 800, 1333) if not plan_flip else (2, 800, 1333)
    frames = torch.from_numpy(bench.synth_frames(B, 3, H, W, 7)).cuda()
    try:
        for name, over in SETTINGS.items():
            cfg = bench.bench_cfg(H, W, 'r50fpn3d')
            _set(cfg, over)
            plan = None
            if plan_flip:
                _set(cfg, {'TEST.COMPETITION_MODE': True, 'TEST.BBOX_AUG.SCORE_HEUR': 'UNION',
                           'TEST.BBOX_AUG.COORD_HEUR': 'UNION', 'TEST.BBOX_AUG.H_FLIP': True})
            blobs, spec = Pm.random_blobs(cfg)
            eng = DetectionEngine(cfg, blobs, spec, dtype='bf16x3')
            if plan_flip:
                plan = tta.view_plan(cfg, spec, H, W)
                assert len(plan.box) == 2
            seen = {}
            inner = eng.box_nms_limit

            def spy(dets, cnt):
                seen['dets'], seen['cnt'] = dets, cnt
                return inner(dets, cnt)
            eng.box_nms_limit = spy
            static_in, run = eng.capture(B, 3, H, W, plan=plan)
            static_in.copy_(frames)
            out = run()
            torch.cuda.synchronize()
            dets_in, cnt_in = seen['dets'].cpu().numpy(), seen['cnt'].cpu().numpy()
            got, gcnt = out['dets'].cpu().numpy(), out['det_counts'].cpu().numpy()
            for b in range(B):
                ref = _oracle_post(cfg, dets_in[b, 0], int(cnt_in[b]))
                assert int(gcnt[b]) == len(ref), (name, b, int(gcnt[b]), len(ref))
                assert np.array_equal(_bits(got[b, 0, :len(ref)]), _bits(ref)), (name, b)
            print('teacher-forced', name, 'flip' if plan_flip else 'plain', 'rows in', cnt_in.tolist(), 'out', gcnt.tolist())
            del eng, run, static_in, out
            torch.cuda.empty_cache()
    finally:
        reset_cfg()


def test_default_step_launches_no_new_kernel():
    """Both options off: the box stage of a detect call makes exactly the parent's library calls."""
    import step_launches as sl
    for wl in ('r50fpn3d', 'r18tube'):
        names = [name for name, _, _ in sl.record((wl, 'bf16x3')).calls]
        assert 'dt_soft_nms_batched' not in names and 'dt_box_vote' not in names
        i = names.index('dt_box_decode')
        tail = [n for n in names[i + 1:] if n in ('dt_nms_batched', 'dt_limit_detections', 'dt_soft_nms_batched', 'dt_box_vote')]
        assert tail[:2] == ['dt_nms_batched', 'dt_limit_detections'], tail


def test_small_clip_soft_linear_vote_meets_parity_rule(monkeypatch):
    """tests/test_gpu_parity_e2e.py's rule on the 96x128 T = 3 clip with SOFT_NMS linear + BBOX_VOTE.  The oracle
    pipeline's box stage is oracle/detections' hard-NMS one; here it runs oracle/soft_nms's stage with the options."""
    from test_gpu_engine import _cfg
    from test_gpu_parity_e2e import _compare
    from detectandtrack_b200.core.config import reset_cfg
    from detectandtrack_b200.modeling import params as Pm
    from oracle import detections as odet
    calls = []

    def stage(*a, **kw):
        calls.append(1)
        return osn.box_results_with_nms_and_limit(*a, soft_nms=('linear', cfg.TEST.SOFT_NMS.SIGMA),
                                                  bbox_vote=cfg.TEST.BBOX_VOTE.VOTE_TH, **kw)
    monkeypatch.setattr(odet, 'box_results_with_nms_and_limit', stage)
    try:
        cfg = _cfg()
        _set(cfg, {'TEST.SOFT_NMS.ENABLED': True, 'TEST.SOFT_NMS.METHOD': 'linear', 'TEST.BBOX_VOTE.ENABLED': True})
        blobs, _ = Pm.random_blobs(cfg, seed=3)
        frames = np.random.RandomState(0).randint(0, 256, (3, 96, 128, 3)).astype(np.uint8)
        r = _compare(cfg, blobs, frames, 'bf16x3')
        assert r['n_det'] > 0 and calls
    finally:
        reset_cfg()
