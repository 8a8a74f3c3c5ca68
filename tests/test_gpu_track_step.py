"""Every tracking launch, bit for bit: the cost kernels (dt_frame_costs, dt_gt_frame_costs), the batched solvers
(dt_lsa_batched on fp32 and fp64 costs, dt_match_frames), the id scan (dt_assign_track_ids) and the prune
(dt_prune_detections) against numpy, scipy and the oracle, at the shapes and edges where they can go wrong.

TABLE lists the launches the engine makes (the tracking leg's shape, every metric set, algo and T, _compute_matches,
_prune_bad_detections and every TRACKING.DEBUG.UPPER_BOUND* mode); each key names the value test that covers it."""
import numpy as np
import pytest
import scipy.optimize

from oracle import keypoints as okp
from oracle import tracking as ot
from oracle.lsa import bipartite_matching_greedy

NAMES = ['nose', 'head_bottom', 'head_top', 'left_ear', 'right_ear', 'left_shoulder', 'right_shoulder', 'left_elbow',
         'right_elbow', 'left_wrist', 'right_wrist', 'left_hip', 'right_hip', 'left_knee', 'right_knee', 'left_ankle', 'right_ankle']
HT, HB = NAMES.index('head_top'), NAMES.index('head_bottom')


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _solve(C, algo):
    """The reference's _compute_matches on a given matrix: matches[q] = p or -1 (scipy for hungarian, its greedy loop)."""
    m = -np.ones(C.shape[1], np.int32)
    if C.shape[0] and C.shape[1]:
        if algo == 'hungarian':
            r, c = scipy.optimize.linear_sum_assignment(C)
        else:
            r, c = bipartite_matching_greedy(C)
        m[np.asarray(c, dtype=np.int64)] = r
    return m


def _ids(matches_per_frame, first_id=0, max_ids=ot.MAX_TRACK_IDS):
    """tracking_engine.py:272-350's id loop over one video's matches."""
    tracks, nxt = [], first_id
    for f, m in enumerate(matches_per_frame):
        ids = []
        for p in m:
            if f == 0 or p == -1:
                ids.append(nxt)
                nxt += 1
                if nxt >= max_ids:
                    nxt %= max_ids
            else:
                ids.append(tracks[f - 1][p])
        tracks.append(ids)
    return tracks


def _ref_cost(prev_b, cur_b, prev_p, cur_p, w_iou, w_pck, names=NAMES):
    """_compute_distance_matrix (tracking_engine.py:158-181): the float32 (1 - IoU) * w and the float64 pck * w of the
    metrics with a non-zero weight, stacked and summed by numpy."""
    Cs = []
    if w_iou:
        Cs.append(ot.distance_matrix(prev_b, cur_b, 1.0) * w_iou)
    if w_pck:
        Cs.append(okp.pairwise_kpt_distance(prev_p, cur_p, names) * w_pck)
    return np.sum(np.stack(Cs, 0), 0)


def _ref_video(frames, poses, w_iou, w_pck, algo='hungarian'):
    ms = [-np.ones(len(frames[0]), np.int32)]
    for f in range(1, len(frames)):
        ms.append(_solve(_ref_cost(frames[f - 1], frames[f], poses[f - 1], poses[f], w_iou, w_pck), algo))
    return ms, _ids(ms)


# ---------------------------------------------------------------------------------------------------- the tie fixture
TIE_WEIGHTS = ((1.0, 0.5), (0.0, 1.0))


def tie_videos(seed=0, n_videos=10, n_frames=31):
    """Crowded frames: 3-14 people with integer box corners in a 300 x 200 region and 17 joints on a quarter grid of each
    box.  The pose-pck costs are multiples of 1/17, so many assignments have equal fp64 total costs that their fp32
    roundings no longer tie."""
    rng = np.random.default_rng(seed)
    videos, vposes = [], []
    for _ in range(n_videos):
        frames, poses = [], []
        for _ in range(n_frames):
            n = int(rng.integers(3, 15))
            x1, y1 = rng.integers(0, 240, n), rng.integers(0, 140, n)
            b = np.stack([x1, y1, x1 + rng.integers(8, 60, n), y1 + rng.integers(8, 60, n), np.ones(n)], 1).astype(np.float32)
            g = rng.integers(0, 5, (2, n, 17)) / 4.0
            px = b[:, 0:1] + g[0] * (b[:, 2:3] - b[:, 0:1])
            py = b[:, 1:2] + g[1] * (b[:, 3:4] - b[:, 1:2])
            p = np.stack([px, py, np.ones_like(px), np.ones_like(px)], 1).astype(np.float32)
            frames.append(b); poses.append([p[i] for i in range(n)])
        videos.append(frames); vposes.append(poses)
    return videos, vposes


def test_tie_fixture_diverges_under_fp32_rounding():
    """The fixture reaches the case the fp64 solve exists for: scipy on the fp64 cost matrix and scipy on its fp32 rounding
    give different assignments for some frame pairs, so the device test below fails on a solver that rounds."""
    videos, vposes = tie_videos()
    diverged = 0
    for w_iou, w_pck in TIE_WEIGHTS:
        for frames, poses in zip(videos, vposes):
            for f in range(1, len(frames)):
                C = _ref_cost(frames[f - 1], frames[f], poses[f - 1], poses[f], w_iou, w_pck)
                assert C.dtype == np.float64
                diverged += not np.array_equal(_solve(C, 'hungarian'), _solve(C.astype(np.float32), 'hungarian'))
    assert diverged >= 2, diverged


@pytest.mark.gpu
@pytest.mark.parametrize('algo', ['hungarian', 'greedy'])
def test_pose_pck_ties_solved_in_fp64(algo):
    """The combined bbox + pose-pck cost is solved as the reference solves it, on the fp64 matrix: the device's matches
    (dt_frame_costs + the batched solver, and _compute_matches on the fp64 matrix) and the engine's track ids equal scipy's
    (or the greedy loop's) on the fp64 sum of the weighted terms."""
    import torch
    from detectandtrack_b200.core import tracking_engine as te
    from detectandtrack_b200.core.config import cfg, reset_cfg
    from detectandtrack_b200.ops import box_ops
    videos, vposes = tie_videos()
    try:
        for w_iou, w_pck in TIE_WEIGHTS:
            reset_cfg()
            cfg.TRACKING.DISTANCE_METRICS = ('bbox-overlap', 'pose-pck')
            cfg.TRACKING.DISTANCE_METRIC_WTS = (w_iou, w_pck)
            cfg.TRACKING.BIPARTITE_MATCHING_ALGO = algo
            got_ids = te._tracks_for_videos(videos, vposes, NAMES)
            flat = [b for v in videos for b in v]
            packed, counts = te._pack(flat)
            is_start = np.zeros(len(flat), np.uint8)
            is_start[np.arange(len(videos)) * len(videos[0])] = 1
            poses = te._pack_poses([p for vp in vposes for p in vp], packed.shape[1], 17)
            d_counts, d_start = _cuda(counts), _cuda(is_start)
            cost = box_ops.frame_costs(_cuda(packed), d_counts, d_start, _cuda(poses), T=1, w_iou=w_iou, w_pck=w_pck,
                                       head_top=HT, head_bottom=HB)
            nrows = torch.cat([d_counts[:1] * 0, d_counts[:-1]]) * (1 - d_start.to(torch.int32))
            m, st = box_ops.lsa_batched(cost, nrows, d_counts, algo)
            m, st = m.cpu().numpy(), st.cpu().numpy()
            assert not st.any()
            f0 = 0
            for v, (frames, poses_v) in enumerate(zip(videos, vposes)):
                ref_m, ref_ids = _ref_video(frames, poses_v, w_iou, w_pck, algo)
                for f in range(1, len(frames)):
                    q = len(frames[f])
                    assert np.array_equal(m[f0 + f, :q], ref_m[f]), (w_iou, w_pck, v, f)
                    if v == 0:
                        C = _ref_cost(frames[f - 1], frames[f], poses_v[f - 1], poses_v[f], w_iou, w_pck)
                        got = te._compute_matches(None, None, None, None, None, None, None, None, algo, C=C)
                        assert np.array_equal(got, ref_m[f]), (w_iou, w_pck, f)
                assert got_ids[v] == ref_ids, (w_iou, w_pck, v)
                f0 += len(frames)
    finally:
        reset_cfg()


# ---------------------------------------------------------------------------------------------------- dt_frame_costs
def _pose(rng, box, K, ht=HT, hb=HB):
    """A [4, K] pose on a quarter grid of the box, with the edges of the pck test: about one pose in four has its head top
    on its head bottom (head size exactly 1)."""
    g = rng.integers(0, 5, (2, K)) / 4.0
    p = np.zeros((4, K), np.float32)
    p[0] = box[0] + g[0] * (box[2] - box[0])
    p[1] = box[1] + g[1] * (box[3] - box[1])
    p[2:] = 1
    if rng.random() < 0.25:
        p[:2, ht] = p[:2, hb]
    return p


def _edge_pair(rng, prev_p, K):
    """A pose of the next frame for prev_p: every joint moved by exactly 0.5 or 0.25 head sizes along x (0.5 is at
    dist_thresh and does not count) or left in place."""
    head = np.float32(np.linalg.norm(prev_p[:2, HT] - prev_p[:2, HB]) + 1)
    p = prev_p.copy()
    p[0] += np.float32(rng.choice([0.0, 0.25, 0.5], K)) * head
    return p


def _cost_frames(rng, T, K, counts, starts):
    """Frames of people for the cost kernels: integer boxes (ties), their T-frame tubes and [4, K] poses, where the
    poses of some people repeat the previous frame's moved by the edge offsets of _edge_pair."""
    frames, poses = [], []
    for f, n in enumerate(counts):
        x1, y1 = rng.integers(0, 240, n), rng.integers(0, 140, n)
        b = np.stack([x1, y1, x1 + rng.integers(8, 60, n), y1 + rng.integers(8, 60, n)], 1).astype(np.float32)
        tube = np.hstack([b + 2 * t for t in range(T)] + [np.ones((n, 1), np.float32)]).astype(np.float32)
        ps = [_pose(rng, b[i], K) for i in range(n)]
        if f and not starts[f] and len(poses[-1]):
            for i in range(min(n, len(poses[-1])) // 2):
                ps[i] = _edge_pair(rng, poses[-1][i], K)
        frames.append(tube); poses.append(ps)
    return frames, poses


@pytest.mark.gpu
@pytest.mark.parametrize('T', [1, 3])
@pytest.mark.parametrize('K', [15, 17])
@pytest.mark.parametrize('w', [(1.0, 0.5), (0.0, 1.0), (1.0, 0.0), (0.5, 2.0)])
def test_frame_costs_exact(T, K, w):
    """dt_frame_costs == np.sum(np.stack([(1 - IoU) * w_iou (float32), pck * w_pck (float64)])) entry by entry over the
    whole [F, dmax, dmax] output: zeros past the counts and on video-start frames, joints exactly at dist_thresh, head
    size 1, K = 15 and 17, w_iou = 0, T = 3."""
    from detectandtrack_b200.core import tracking_engine as te
    from detectandtrack_b200.ops import box_ops
    w_iou, w_pck = w
    rng = np.random.default_rng(100 * T + K)
    counts = [9, 14, 0, 5, 14, 1, 12, 12, 3]
    starts = [1, 0, 0, 0, 1, 0, 0, 1, 0]
    dmax = 16                                                         # > every count: the padding is written too
    frames, poses = _cost_frames(rng, T, K, counts, starts)
    packed, cnt = te._pack(frames)
    packed = np.concatenate([packed, np.zeros((len(frames), dmax - packed.shape[1], packed.shape[2]), np.float32)], 1)
    pp = te._pack_poses(poses, dmax, K)
    cost = box_ops.frame_costs(_cuda(packed), _cuda(cnt), _cuda(np.array(starts, np.uint8)), _cuda(pp), T=T, w_iou=w_iou,
                               w_pck=w_pck, head_top=HT, head_bottom=HB).cpu().numpy()
    assert cost.dtype == np.float64 and cost.shape == (len(frames), dmax, dmax)
    names = NAMES[:K]
    for f in range(len(frames)):
        ref = np.zeros((dmax, dmax))
        if not starts[f]:
            P, Q = counts[f - 1], counts[f]
            if P and Q:
                ref[:P, :Q] = _ref_cost(frames[f - 1], frames[f], poses[f - 1], poses[f], w_iou, w_pck, names)
        assert np.array_equal(cost[f], ref), (f, np.argwhere(cost[f] != ref)[:4])
    if w_pck:                                                         # the edges were reached
        assert any(np.any(np.linalg.norm(p[:2, HT] - p[:2, HB]) == 0) for ps in poses for p in ps)


@pytest.mark.gpu
@pytest.mark.parametrize('w', [(1.0, 1.0), (0.0, 1.0), (1.0, 0.0)])
def test_gt_frame_costs_exact(w):
    """dt_gt_frame_costs == the reference's matrix with the frame's GT as the previous frame: float32 (1 - IoU) * w_iou and
    the pck of the int32 GT keypoints (numpy promotes them and the fp32 detections to fp64) * w_pck, summed in fp64; GT
    heads of size 1, joints exactly half a head away, zeros past the counts."""
    from detectandtrack_b200.ops import box_ops
    w_iou, w_pck = w
    rng = np.random.default_rng(7)
    K, R, dmax = 17, 4, 12
    gcounts, dcounts = [5, 0, 11, 3, 12], [7, 4, 0, 12, 1]
    F = len(gcounts)
    pb = np.zeros((2 * F, dmax, 5), np.float32)
    pp = np.zeros((2 * F, dmax, R, K), np.float32)
    cnt = np.zeros(2 * F, np.int32)
    gts, dts = [], []
    for f in range(F):
        G, n = gcounts[f], dcounts[f]
        x1, y1 = rng.integers(0, 240, G), rng.integers(0, 140, G)
        gb = np.stack([x1, y1, x1 + rng.integers(8, 60, G), y1 + rng.integers(8, 60, G)], 1).astype(np.float32)
        gk = np.zeros((G, 3, K), np.int32)
        gk[:, 0] = x1[:, None] + rng.integers(0, 9, (G, K)); gk[:, 1] = y1[:, None] + rng.integers(0, 9, (G, K)); gk[:, 2] = 2
        gk[::3, :2, HT] = gk[::3, :2, HB]                                # head size 1
        db = np.hstack([gb[rng.integers(0, max(G, 1), n)] + rng.integers(-3, 4, (n, 4)) if G else
                        rng.integers(0, 200, (n, 4)).astype(np.float32), np.ones((n, 1))]).astype(np.float32)
        dp = np.zeros((n, R, K), np.float32)
        src = rng.integers(0, max(G, 1), n)
        for i in range(n):
            if G:
                head = np.linalg.norm(gk[src[i], :2, HT] - gk[src[i], :2, HB]).astype(np.float64) + 1
                dp[i, :2] = gk[src[i], :2] + np.float32(rng.choice([0.0, 0.5, 0.75], K)) * np.float32(head) * np.array([[1], [0]])
            dp[i, 2:] = rng.random((2, K))
        pb[2 * f, :G, :4] = gb; pp[2 * f, :G, :3] = gk
        pb[2 * f + 1, :n] = db; pp[2 * f + 1, :n] = dp
        cnt[2 * f], cnt[2 * f + 1] = G, n
        gts.append((gb, gk)); dts.append((db, dp))
    cost = box_ops.gt_frame_costs(_cuda(pb), _cuda(cnt), _cuda(pp), T=1, w_iou=w_iou, w_pck=w_pck, head_top=HT,
                                  head_bottom=HB).cpu().numpy()
    assert cost.dtype == np.float64
    for f in range(F):
        (gb, gk), (db, dp) = gts[f], dts[f]
        ref = np.zeros((dmax, dmax))
        if len(gb) and len(db):
            gpad = np.hstack([gb, np.zeros((len(gb), 1), np.float32)])
            ref[:len(gb), :len(db)] = _ref_cost(gpad, db, list(gk), list(dp), w_iou, w_pck)
        assert np.array_equal(cost[f], ref), (f, np.argwhere(cost[f] != ref)[:4])


# ---------------------------------------------------------------------------------------------------- dt_match_frames
def leg_videos():
    """bench.tracking_leg's two variants (64 videos x 30 frames x 100 detections each, seed 3): tie-heavy, then the same
    generator with sub-pixel jitter (tie-free)."""
    out = []
    for tie_free in (False, True):
        rng = np.random.default_rng(3)
        vids = [ot.synth_video(rng, n_frames=30, n_dets=100) for _ in range(64)]
        if tie_free:
            vids = [[(f + np.concatenate([rng.uniform(0, 1e-2, (f.shape[0], 4)), np.zeros((f.shape[0], 1))], 1)).astype(np.float32)
                     for f in v] for v in vids]
        out += vids
    return out


@pytest.mark.gpu
def test_match_frames_leg_shape():
    """The tracking leg in one launch: both variants (128 videos, 3840 frames, is_start every 30 frames); the ids of every
    video equal the reference loop's with scipy."""
    from detectandtrack_b200.core import tracking_engine as te
    from detectandtrack_b200.core.config import reset_cfg
    reset_cfg()
    vids = leg_videos()
    got = te._tracks_for_videos(vids)
    for v, frames in enumerate(vids):
        assert got[v] == [[int(x) for x in t] for t in ot.compute_tracks_video(frames, solver='scipy')], v


def _degenerate_frames(rng, T, counts):
    """Boxes at the IoU kernel's edges, against the previous frame: an identical box, a box whose '+1' overlap with one is
    exactly 0, boxes of '+1' width 0 and of negative width, on integer corners so that many costs tie."""
    frames = []
    for n in counts:
        x1, y1 = rng.integers(0, 120, (n, T)).astype(np.float32), rng.integers(0, 80, (n, T)).astype(np.float32)
        wd, ht = rng.integers(-2, 40, (n, T)).astype(np.float32), rng.integers(-2, 40, (n, T)).astype(np.float32)
        b = np.stack([x1, y1, x1 + wd, y1 + ht], 2)                       # [n, T, 4]
        prev = frames[-1][:, :4 * T].reshape(-1, T, 4) if frames else np.zeros((0, T, 4), np.float32)
        if n >= 4 and len(prev) >= 2:
            b[0] = prev[0]                                                 # identical
            b[1, :, 0] = prev[1, :, 2] + 1; b[1, :, 2] = b[1, :, 0] + 19  # min(x2) - max(x1) + 1 == 0
            b[1, :, 1], b[1, :, 3] = prev[1, :, 1], prev[1, :, 3]
            b[2, :, 2] = b[2, :, 0] - 1                                    # '+1' width 0
            b[3, :, 2] = b[3, :, 0] - 6                                    # negative width
        frames.append(np.hstack([b.reshape(n, 4 * T), rng.random((n, 1))]).astype(np.float32))
    return frames


@pytest.mark.gpu
@pytest.mark.parametrize('algo', ['hungarian', 'greedy'])
@pytest.mark.parametrize('T', [1, 3, 8])
def test_match_frames_edges(T, algo):
    """dt_match_frames against the reference's (1 - IoU) * weight solved by scipy / the greedy loop: T up to DT_MAX_T,
    rows padded past 4T + 1, weight 0.5, degenerate boxes, counts 0, 1 and dmax, with and without is_start."""
    from detectandtrack_b200.ops import box_ops
    rng = np.random.default_rng(T)
    dmax = 37
    counts = [dmax, 0, 1, dmax, 1, 20, dmax, dmax, 5, 0, 9, dmax]
    starts = np.array([1, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0], np.uint8)
    frames = _degenerate_frames(rng, T, counts)
    ld = 4 * T + 1 + 3
    packed = np.zeros((len(frames), dmax, ld), np.float32)
    for f, b in enumerate(frames):
        packed[f, :len(b), :4 * T + 1] = b
        packed[f, :len(b), 4 * T + 1:] = np.nan                           # never read
    for weight in (1.0, 0.5):
        for start in (starts, None):
            m = box_ops.match_frames(_cuda(packed), _cuda(np.array(counts, np.int32)), None if start is None else _cuda(start),
                                     T=T, weight=weight, algo=algo)[0].cpu().numpy()
            for f in range(len(frames)):
                Q = counts[f]
                if f == 0 or (start is not None and start[f]):
                    ref = -np.ones(Q, np.int32)
                else:
                    ref = _solve(ot.distance_matrix(frames[f - 1], frames[f], weight), algo) if counts[f - 1] else -np.ones(Q, np.int32)
                assert np.array_equal(m[f, :Q], ref), (weight, start is None, f)
                assert np.all(m[f, Q:] == -1)


# ---------------------------------------------------------------------------------------------------- dt_lsa_batched(_f64)
def _lsa_launch(cost, nr, nc, algo, ldc):
    """dt_lsa_batched / dt_lsa_batched_f64 (by the cost's dtype) on cost [B, dmax, dmax] laid out with row stride ldc."""
    import torch
    from detectandtrack_b200 import _lib as L
    from detectandtrack_b200.ops import box_ops
    B, dmax, _ = cost.shape
    wide = np.full((B, dmax, ldc), np.nan, cost.dtype)                # columns past dmax are never read
    wide[:, :, :dmax] = cost
    d, d_nr, d_nc = _cuda(wide), _cuda(np.asarray(nr, np.int32)), _cuda(np.asarray(nc, np.int32))
    m = torch.empty((B, dmax), dtype=torch.int32, device='cuda')
    st = torch.empty((B,), dtype=torch.int32, device='cuda')
    name = 'dt_lsa_batched_f64' if cost.dtype == np.float64 else 'dt_lsa_batched'
    L.call(name, L.ptr(d), B, dmax, ldc, L.ptr(d_nr), L.ptr(d_nc), box_ops.ALGOS[algo], L.ptr(m), L.ptr(st), L.stream_ptr())
    return m.cpu().numpy(), st.cpu().numpy()


def _tie_costs(rng, P, Q, kind, dtype):
    if kind == 0:
        C = rng.random((P, Q))
    elif kind == 1:
        C = rng.integers(0, 3, (P, Q)).astype(np.float64)
    elif kind == 2:
        C = np.ones((P, Q)); msk = rng.random((P, Q)) < 0.1; C[msk] = rng.random(int(msk.sum()))
    else:
        C = 1.0 - rng.integers(0, 18, (P, Q)) / 17.0                     # pose-pck-like sixteenths of ties
    return C.astype(dtype)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [np.float32, np.float64])
@pytest.mark.parametrize('algo', ['hungarian', 'greedy'])
def test_lsa_batched_shapes(dtype, algo):
    """Both solvers against scipy / the greedy loop: dmax 1, 33, 100, 223 and 224 with ldc > dmax, random P x Q up to
    dmax, the extreme rectangles 1 x 224 and 224 x 1 (the transposed path), 224 x 223, and the tie-heavy costs of the
    tracker (all-ones with a few values, small integers, multiples of 1/17)."""
    rng = np.random.default_rng(5 if dtype == np.float32 else 6)
    for dmax in (1, 33, 100, 223, 224):
        shapes = [(int(rng.integers(0, dmax + 1)), int(rng.integers(0, dmax + 1))) for _ in range(8)] + [(dmax, dmax)]
        if dmax == 224:
            shapes += [(1, 224), (224, 1), (224, 223), (223, 224)]
        if algo == 'greedy' and dmax >= 223:
            shapes = shapes[-4:]                                           # the greedy loop's np.delete is slow at 224
        cost = np.zeros((len(shapes), dmax, dmax), dtype)
        for b, (P, Q) in enumerate(shapes):
            cost[b, :P, :Q] = _tie_costs(rng, P, Q, b % 4, dtype)
        nr, nc = [s[0] for s in shapes], [s[1] for s in shapes]
        m, st = _lsa_launch(cost, nr, nc, algo, dmax + 5)
        assert not st.any(), dmax
        for b, (P, Q) in enumerate(shapes):
            assert np.array_equal(m[b, :Q], _solve(cost[b, :P, :Q], algo)), (dmax, P, Q)
            assert np.all(m[b, Q:] == -1)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [np.float32, np.float64])
def test_lsa_nonfinite_costs_report_status(dtype):
    """A NaN entry, a -inf entry and a row that is all +inf: scipy raises ValueError; the Hungarian solver returns status 1
    for those problems (and solves the finite one beside them), and the engine raises ValueError like scipy."""
    from detectandtrack_b200.core import tracking_engine as te
    from detectandtrack_b200.core.config import cfg, reset_cfg
    rng = np.random.default_rng(9)
    bad = []
    C = rng.random((5, 6)); C[2, 3] = np.nan; bad.append(C)
    C = rng.random((6, 4)); C[4, 0] = -np.inf; bad.append(C)
    C = rng.random((4, 4)); C[1] = np.inf; bad.append(C)
    for C in bad:
        with pytest.raises(ValueError):
            scipy.optimize.linear_sum_assignment(C.astype(dtype))
    ok = rng.random((6, 6))
    cost = np.zeros((4, 6, 6), dtype)
    for b, C in enumerate(bad + [ok]):
        cost[b, :C.shape[0], :C.shape[1]] = C
    m, st = _lsa_launch(cost, [5, 6, 4, 6], [6, 4, 4, 6], 'hungarian', 6)
    assert st.tolist() == [1, 1, 1, 0]
    assert np.array_equal(m[3], _solve(cost[3], 'hungarian'))
    for C in bad:
        with pytest.raises(ValueError):
            te._compute_matches(None, None, None, None, None, None, None, None, 'hungarian', C=C.astype(dtype))
    if dtype == np.float64:                                            # an infinite weight: inf * 0 = NaN in the matrix
        videos, vposes = tie_videos(n_videos=1, n_frames=3)
        try:
            reset_cfg()
            cfg.TRACKING.DISTANCE_METRICS = ('bbox-overlap', 'pose-pck')
            cfg.TRACKING.DISTANCE_METRIC_WTS = (1.0, float('inf'))
            with pytest.raises(ValueError):
                _ref_video(videos[0], vposes[0], 1.0, np.inf)
            with pytest.raises(ValueError):
                te._tracks_for_videos(videos, vposes, NAMES)
        finally:
            reset_cfg()


# ---------------------------------------------------------------------------------------------------- dt_assign_track_ids
def _random_matches(rng, P, Q):
    m = -np.ones(Q, np.int32)
    k = min(P, Q, int(rng.integers(0, min(P, Q) + 1)))
    m[rng.choice(Q, k, replace=False)] = rng.choice(P, k, replace=False)
    return m


@pytest.mark.gpu
@pytest.mark.parametrize('first_id,max_ids', [(0, 999), (5, 999), (3, 50)])
def test_assign_track_ids_wrap(first_id, max_ids):
    """Several videos in one launch, each restarting at first_id: one whose counts alternate 100, 0, 100, ... over 22
    frames (1100 new ids: they wrap at MAX_TRACK_IDS), one with an empty frame inside, one of a single frame; ids equal the
    reference's loop with its wrap rule (next_id %= max_ids once it reaches max_ids)."""
    from detectandtrack_b200.ops import box_ops
    rng = np.random.default_rng(first_id + max_ids)
    dmax = 100
    videos = [[100 if f % 2 == 0 else 0 for f in range(22)], [30, 41, 0, 17, 100, 99, 3], [8],
              [int(rng.integers(0, 101)) for _ in range(15)]]
    counts, mats, first, per_video = [], [], [], []
    for vc in videos:
        first.append(len(counts))
        ms = []
        for f, n in enumerate(vc):
            m = rng.integers(-1, dmax, n).astype(np.int32) if f == 0 else _random_matches(rng, vc[f - 1], n)
            ms.append(m)                                                   # a video's first frame: never read
            row = np.full(dmax, 7, np.int32); row[:n] = m
            mats.append(row); counts.append(n)
        per_video.append(ms)
    is_start = np.zeros(len(counts), np.uint8); is_start[first] = 1
    tr = box_ops.assign_track_ids(_cuda(np.stack(mats)), _cuda(np.array(counts, np.int32)),
                                  _cuda(np.array(first, np.int32)), _cuda(is_start), first_id, max_ids).cpu().numpy()
    for v, ms in enumerate(per_video):
        ref = _ids(ms, first_id, max_ids)
        for f, ids in enumerate(ref):
            g = first[v] + f
            assert tr[g, :counts[g]].tolist() == ids, (v, f)
            assert np.all(tr[g, counts[g]:] == -1)
    assert sum(videos[0]) > ot.MAX_TRACK_IDS


# ---------------------------------------------------------------------------------------------------- dt_prune_detections
@pytest.mark.gpu
@pytest.mark.parametrize('T', [1, 3])
@pytest.mark.parametrize('center_only', [0, 1])
def test_prune_detections(T, center_only):
    """dt_prune_detections == ot.center_boxes / ot.prune_boxes: 127 to 300 rows per frame (the compaction's carry across
    128-row passes), scores exactly at conf and NaN, clipped areas exactly at min_area, boxes half outside the image,
    rows padded past 4T + 1."""
    from detectandtrack_b200.ops import box_ops
    rng = np.random.default_rng(10 * T + center_only)
    dmax, conf, H, W = 300, np.float32(0.95), 240, 320
    ns = [127, 128, 129, 255, 256, 300, 0, 1]
    ld = 4 * T + 1 + 2
    packed = np.zeros((len(ns), dmax, ld), np.float32)
    frames = []
    for f, n in enumerate(ns):
        x1, y1 = rng.integers(-40, W, (n, T)).astype(np.float32), rng.integers(-40, H, (n, T)).astype(np.float32)
        w, h = rng.integers(0, 60, (n, T)).astype(np.float32), rng.integers(0, 60, (n, T)).astype(np.float32)
        b = np.stack([x1, y1, x1 + w, y1 + h], 2).reshape(n, 4 * T)
        sc = rng.choice(np.array([0.5, 0.94, 0.95, 0.96, 1.0, np.nan], np.float32), n)
        c = T // 2 if center_only else 0
        for i in range(0, n, 7):                                           # clipped area exactly 50: [-3, 5] x [y, y + 10]
            b[i, 4 * c:4 * c + 4] = [-3, 20, 5, 30]
        for i in range(3, n, 11):                                          # half outside on the right
            b[i, 4 * c:4 * c + 4] = [W - 10, 40, W + 10, 60]
        rows = np.hstack([b, sc[:, None]]).astype(np.float32)
        frames.append(rows)
        packed[f, :n, :4 * T + 1] = rows
        packed[f, :n, 4 * T + 1:] = -7
    hw = np.tile(np.array([[H, W]], np.float32), (len(ns), 1))
    out, cnt, sel = box_ops.prune_detections(_cuda(packed), _cuda(np.array(ns, np.int32)), _cuda(hw), float(conf), T=T,
                                             center_only=bool(center_only), min_area=50.0)
    out, cnt, sel = out.cpu().numpy(), cnt.cpu().numpy(), sel.cpu().numpy()
    To = 1 if center_only else T
    carried = 0
    for f, rows in enumerate(frames):
        c = ot.center_boxes(rows.copy()) if center_only else rows.copy()
        keep = ot.prune_boxes(c, H, W, conf) if len(c) else np.zeros(0, np.int64)
        n = len(keep)
        assert cnt[f] == n, f
        assert np.array_equal(sel[f, :n], keep), f
        assert np.array_equal(out[f, :n], c[keep].reshape(n, 4 * To + 1)), f
        carried += bool(n) and keep.min() < 128 <= keep.max()         # rows kept in both 128-row passes
    assert carried >= 3, carried


# ---------------------------------------------------------------------------------------------------- launch table
# key: (entry point, algo, T, w_iou != 0, w_pck != 0, is_start given, center_only); None where the entry point has no such
# argument.  Value: the test above that checks launches of that key.
H, G = 'hungarian', 'greedy'
TABLE = {
    ('dt_match_frames', H, 1, True, None, True, None): 'test_match_frames_leg_shape',
    ('dt_match_frames', G, 1, True, None, True, None): 'test_match_frames_edges',
    ('dt_match_frames', H, 3, True, None, True, None): 'test_match_frames_edges',
    ('dt_match_frames', G, 3, True, None, True, None): 'test_match_frames_edges',
    ('dt_match_frames', H, 1, True, None, False, None): 'test_match_frames_edges',
    ('dt_match_frames', G, 1, True, None, False, None): 'test_match_frames_edges',
    ('dt_match_frames', H, 3, True, None, False, None): 'test_match_frames_edges',
    ('dt_match_frames', G, 3, True, None, False, None): 'test_match_frames_edges',
    ('dt_frame_costs', None, 1, True, True, True, None): 'test_frame_costs_exact',
    ('dt_frame_costs', None, 3, True, True, True, None): 'test_frame_costs_exact',
    ('dt_frame_costs', None, 1, False, True, True, None): 'test_frame_costs_exact',
    ('dt_frame_costs', None, 3, False, True, True, None): 'test_frame_costs_exact',
    ('dt_gt_frame_costs', None, 1, True, True, None, None): 'test_gt_frame_costs_exact',
    ('dt_lsa_batched', H, None, None, None, None, None): 'test_lsa_batched_shapes',
    ('dt_lsa_batched', G, None, None, None, None, None): 'test_lsa_batched_shapes',
    ('dt_lsa_batched_f64', H, None, None, None, None, None): 'test_pose_pck_ties_solved_in_fp64',
    ('dt_lsa_batched_f64', G, None, None, None, None, None): 'test_pose_pck_ties_solved_in_fp64',
    ('dt_assign_track_ids', None, None, None, None, True, None): 'test_assign_track_ids_wrap',
    ('dt_prune_detections', None, 1, None, None, None, 0): 'test_prune_detections',
    ('dt_prune_detections', None, 3, None, None, None, 0): 'test_prune_detections',
}


def launch_key(name, a):
    """The table key of one L.call(name, *a) of the tracking entry points, or None for other entry points
    (dt_track_upper_bound's row copies are checked against the reference's goldens in test_gpu_upper_bound.py)."""
    if name in ('dt_lsa_batched', 'dt_lsa_batched_f64'):
        return (name, (H, G)[a[6]], None, None, None, None, None)
    if name == 'dt_match_frames':
        return (name, (H, G)[a[8]], a[4], a[7] != 0, None, a[6] is not None, None)
    if name == 'dt_frame_costs':
        return (name, None, a[2], a[13] != 0, a[14] != 0, a[10] is not None, None)
    if name == 'dt_gt_frame_costs':
        return (name, None, a[2], a[12] != 0, a[13] != 0, None, None)
    if name == 'dt_assign_track_ids':
        return (name, None, None, None, None, a[2] is not None, None)
    if name == 'dt_prune_detections':
        return (name, None, a[4], None, None, None, a[5])
    return None


def _engine_set(rng, T, n_videos=2, n_frames=4):
    """json_data and dets of a few small videos (5-12 people, a [4, 17] pose each, the GT the roidb holds for the
    upper-bound modes), for compute_matches_tracks."""
    json_data, boxes, poses = [], [], []
    for v in range(n_videos):
        for f in range(n_frames):
            n = int(rng.integers(5, 13))
            x1, y1 = rng.integers(0, 240, n), rng.integers(0, 140, n)
            b = np.stack([x1, y1, x1 + rng.integers(8, 60, n), y1 + rng.integers(8, 60, n)], 1).astype(np.float32)
            kp = np.zeros((n, 3, 17), np.int32)
            kp[:, 0] = b[:, :1] + rng.integers(0, 8, (n, 17)); kp[:, 1] = b[:, 1:2] + rng.integers(0, 8, (n, 17)); kp[:, 2] = 2
            json_data.append({'image': 'vid%02d/%06d.jpg' % (v, f), 'height': 240, 'width': 320, 'boxes': np.tile(b, (1, T)),
                              'gt_keypoints': kp, 'tracks': np.arange(n) + 100 * v})
            db = np.hstack([np.tile(b + rng.integers(-3, 4, b.shape), (1, T)), rng.uniform(0.9, 1, (n, 1))]).astype(np.float32)
            p = np.zeros((n, 4, 17), np.float32)
            p[:, :3] = kp + rng.integers(-2, 3, kp.shape)
            boxes.append(db); poses.append([p[i] for i in range(n)])
    return json_data, boxes, poses


@pytest.mark.gpu
def test_tracking_launches_are_all_in_the_table(monkeypatch):
    """Every launch of the tracking entry points made by the tracking leg, compute_matches_tracks with each metric set
    (bbox, bbox + pose-pck, pose-pck), algo and T, _compute_matches with and without C, _prune_bad_detections and every
    TRACKING.DEBUG.UPPER_BOUND* mode has a key in TABLE; every key was launched and names a value test of this file."""
    import copy
    from detectandtrack_b200 import _lib as L
    from detectandtrack_b200.core import tracking_engine as te
    from detectandtrack_b200.core.config import cfg, reset_cfg
    launched = set()
    orig_call = L.call

    def spy(name, *a):
        k = launch_key(name, a)
        if k is not None:
            launched.add(k)
        return orig_call(name, *a)
    monkeypatch.setattr(L, 'call', spy)
    rng = np.random.default_rng(12)
    try:
        reset_cfg()
        te._tracks_for_videos([ot.synth_video(np.random.default_rng(3), n_frames=30, n_dets=100) for _ in range(64)])
        for T in (1, 3):
            json_data, boxes, poses = _engine_set(rng, T)
            mk = lambda: {'all_boxes': [[], [b.copy() for b in boxes]], 'all_keyps': [[], [list(p) for p in poses]]}
            for metrics in ((1.0, 0.0), (1.0, 0.5), (0.0, 1.0)):
                for algo in (H, G):
                    reset_cfg()
                    cfg.TRACKING.DISTANCE_METRICS = ('bbox-overlap', 'pose-pck')
                    cfg.TRACKING.DISTANCE_METRIC_WTS = metrics
                    cfg.TRACKING.BIPARTITE_MATCHING_ALGO = algo
                    te.compute_matches_tracks(json_data, mk())
            reset_cfg()
            for algo in (H, G):
                te._compute_matches(None, None, boxes[0], boxes[1], None, None, ('bbox-overlap',), (1.0,), algo)
                C = rng.random((5, 7))
                te._compute_matches(None, None, None, None, None, None, None, None, algo, C=C.astype(np.float32))
                te._compute_matches(None, None, None, None, None, None, None, None, algo, C=C)
            te._prune_bad_detections(mk(), json_data, 0.95)
        json_data, boxes, poses = _engine_set(rng, 1)
        modes = ((1, 0, 0, 0), (1, 1, 0, 0), (1, 1, 1, 0), (0, 0, 0, 1), (1, 0, 0, 1))
        for ub, ub2, conf, ub5 in modes:
            for w_pck in (0.0, 1.0):
                for algo in (H, G):
                    reset_cfg()
                    d = cfg.TRACKING.DEBUG
                    d.UPPER_BOUND, d.UPPER_BOUND_2_GT_KPS, d.UPPER_BOUND_2_GT_KPS_ONLY_CONF, d.UPPER_BOUND_5_GT_KPS_ONLY = \
                        bool(ub), bool(ub2), bool(conf), bool(ub5)
                    cfg.TRACKING.DISTANCE_METRICS = ('bbox-overlap', 'pose-pck')
                    cfg.TRACKING.DISTANCE_METRIC_WTS = (1.0, w_pck)
                    cfg.TRACKING.BIPARTITE_MATCHING_ALGO = algo
                    te.compute_matches_tracks(copy.deepcopy(json_data), {'all_boxes': [[], [b.copy() for b in boxes]],
                                                                         'all_keyps': [[], [list(p) for p in poses]]})
    finally:
        reset_cfg()
    assert launched - set(TABLE) == set(), sorted(launched - set(TABLE), key=str)
    assert set(TABLE) - launched == set(), sorted(set(TABLE) - launched, key=str)
    for k, test in TABLE.items():
        assert test.startswith('test_') and callable(globals().get(test)), (k, test)
