"""PoseTrack evaluation: poseval's ``evaluate_simple.evaluate`` (lib/datasets/posetrack/poseval/py/) with the frame
assignment, the per-joint AP and the CLEAR-MOT accumulation on the device (csrc/poseval.cu).

    evaluate(gtdir, preddir, eval_pose=True, eval_track=True, eval_upper_bound=False) -> ((apAll, preAll, recAll), metrics)
    evaluate_upper_bound(gtdir, preddir, ...)       the same with poseval's upper-bound MOT (eval_helpers.py:559-573)

The host part restates ``eval_helpers.load_data_dir`` + ``cleanupData`` + ``removeIgnoredPoints`` (eval_helpers.py:282-415)
and packs the result into flat fp64 arrays (``PoseTrackPack``).  Everything after that (distances, PCK, the GT/prediction
assignment, the sort and RPC scan of every joint, MOTAccumulator.update of every (sequence, joint)) runs in three device
launches; only the reference's final per-joint arithmetic (evaluateAP.py:28-30, evaluateTracking.py:108-133) is done in
numpy on the 15 per-joint sums, exactly as the reference writes it.

Choices where the reference is not deterministic or not portable:
  - GT files are read in sorted name order (the reference takes glob order, i.e. whatever the directory lists).  The order
    decides the track-id offsets, which frame a stale MOT input comes from (below) and the last bits of sumD.
  - Scores that tie are ranked by their position in the reference's concatenation order (frame, then prediction).  The
    reference's ``np.argsort(scores)[::-1]`` leaves ties to numpy's unstable sort; AP does not depend on the order inside
    a tie group whose labels are all equal (the writer's -100 dummy joints are such a group).
  - Ignore regions use an exact point-in-polygon test (a point on the boundary is not inside, like shapely's
    ``Polygon.contains``): a floating-point orientation test with Shewchuk's error bound, exact rationals where it cannot
    decide.  A region of fewer than 3 points raises ValueError, as shapely's LinearRing does.
  - The reference's ``motAll[imgidx]`` is filled from ``if 'mot' in locals()``: a frame without both GT and predictions
    reuses the MOT inputs of the previous such frame in global frame order, even from another sequence.  That is kept.
    When no earlier frame has MOT inputs the reference fails (an assertion in computeMetrics); here that is a ValueError
    naming the frame.
"""
import glob
import json
import os.path as osp
from fractions import Fraction

import numpy as np

from .. import _lib as L

N_JOINTS = 15
MAX_TRACK_ID = 1000

# eval_helpers.Joint
RIGHT_ANKLE, RIGHT_KNEE, RIGHT_HIP, LEFT_HIP, LEFT_KNEE, LEFT_ANKLE, RIGHT_WRIST, RIGHT_ELBOW, RIGHT_SHOULDER, \
    LEFT_SHOULDER, LEFT_ELBOW, LEFT_WRIST, NECK, NOSE, HEAD_TOP = range(N_JOINTS)


# ---- ignore regions ---------------------------------------------------------------------------------------------------

_U = np.finfo(np.float64).eps / 2
_CCW_ERRBOUND = (3.0 + 16.0 * _U) * _U             # Shewchuk's ccwerrboundA


def _orient_sign(ax, ay, bx, by, px, py):
    """Exact sign of orient2d(a, b, p) (> 0: p left of a -> b), arrays broadcast."""
    l = (ax - px) * (by - py)
    r = (ay - py) * (bx - px)
    det = l - r
    sign = np.sign(det).astype(np.int64)
    unsure = ~(np.abs(det) > _CCW_ERRBOUND * (np.abs(l) + np.abs(r)))
    if unsure.any():
        A = np.broadcast_arrays(ax, ay, bx, by, px, py)
        for idx in zip(*np.nonzero(unsure)):
            a_x, a_y, b_x, b_y, p_x, p_y = (Fraction(float(v[idx])) for v in A)
            d = (a_x - p_x) * (b_y - p_y) - (a_y - p_y) * (b_x - p_x)
            sign[idx] = (d > 0) - (d < 0)
    return sign


def polygon_contains(poly, pts):
    """shapely ``Polygon(poly).contains(Point(p))`` for every p of pts [n, 2]: strictly inside (even-odd rule), a point on
    an edge or a vertex is not contained.  poly: [m, 2], m >= 3 (ValueError otherwise)."""
    poly = np.asarray(poly, np.float64).reshape(-1, 2)
    if len(poly) < 3:
        raise ValueError('A LinearRing must have at least 3 coordinate tuples (ignore region with %d points)' % len(poly))
    pts = np.asarray(pts, np.float64).reshape(-1, 2)
    if len(pts) == 0:
        return np.zeros(0, bool)
    a, b = poly, np.roll(poly, -1, axis=0)
    ax, ay, bx, by = (v[None, :] for v in (a[:, 0], a[:, 1], b[:, 0], b[:, 1]))
    px, py = pts[:, 0:1], pts[:, 1:2]
    s = _orient_sign(ax, ay, bx, by, px, py)
    on_edge = (s == 0) & (np.minimum(ax, bx) <= px) & (px <= np.maximum(ax, bx)) & \
        (np.minimum(ay, by) <= py) & (py <= np.maximum(ay, by))
    crosses = ((ay > py) != (by > py)) & np.where(by > ay, s > 0, s < 0)
    return ~on_edge.any(axis=1) & (crosses.sum(axis=1) % 2 == 1)


# ---- eval_helpers.load_data_dir ---------------------------------------------------------------------------------------

def _rect_has_points(rect):
    return (('annopoints' in rect.keys()) and (len(rect['annopoints']) > 0 and len(rect['annopoints'][0]) > 0) and
            ('point' in rect['annopoints'][0].keys()))


def _remove_rects_without_points(rects):
    return [r for r in rects if _rect_has_points(r)]


def _remove_ignored_points_rects(rects, polys):
    out = []
    for rect in rects:
        points = rect['annopoints'][0]['point']
        if polys and points:
            xy = np.array([[p['x'][0], p['y'][0]] for p in points], np.float64)
            ignored = np.zeros(len(points), bool)
            for poly in polys:
                ignored |= polygon_contains(poly, xy)
            points = [p for p, ig in zip(points, ignored) if not ig]
        if len(points) > 0:
            rect['annopoints'][0]['point'] = points
            out.append(rect)
    return out


def _offset_track_ids(frames, i, what):
    for frame in frames:
        for rect in frame['annorect']:
            if 'track_id' in rect.keys():
                if not rect['track_id'][0] < MAX_TRACK_ID:
                    raise ValueError('%s track id %s >= %d (MAX_TRACK_ID)' % (what, rect['track_id'][0], MAX_TRACK_ID))
                rect['track_id'][0] += i * MAX_TRACK_ID


def load_data_dir(gt_dir, pred_dir):
    """eval_helpers.load_data_dir: (gtFramesAll, prFramesAll, gt file names), GT files in sorted order."""
    if not osp.exists(gt_dir):
        raise IOError('Given GT directory ' + gt_dir + ' does not exist!')
    if not osp.exists(pred_dir):
        raise IOError('Given prediction directory ' + pred_dir + ' does not exist!')
    filenames = sorted(glob.glob(osp.join(gt_dir, '*.json')))
    gtFramesAll, prFramesAll = [], []
    for i, fname in enumerate(filenames):
        with open(fname) as fin:
            gt = json.load(fin)['annolist']
        for frame in gt:
            frame['seq_id'] = i
        _offset_track_ids(gt, i, 'GT')
        gtFramesAll += gt
        pred_fname = osp.join(pred_dir, osp.basename(fname))
        if not osp.exists(pred_fname):
            raise IOError('Prediction file ' + pred_fname + ' does not exist')
        with open(pred_fname) as fin:
            pr = json.load(fin)['annolist']
        if len(pr) != len(gt):
            raise ValueError('# prediction frames %d <> # GT frames %d for %s' % (len(pr), len(gt), pred_fname))
        _offset_track_ids(pr, i, 'prediction')
        prFramesAll += pr
    # cleanupData: drop GT frames without rects (and their predictions), then the rects without points
    keep = [k for k in range(len(gtFramesAll)) if len(gtFramesAll[k]['annorect']) > 0]
    gtFramesAll = [gtFramesAll[k] for k in keep]
    prFramesAll = [prFramesAll[k] for k in keep]
    for gtf, prf in zip(gtFramesAll, prFramesAll):
        gtf['annorect'] = _remove_rects_without_points(gtf['annorect'])
        prf['annorect'] = _remove_rects_without_points(prf['annorect'])
    # removeIgnoredPoints
    for gtf, prf in zip(gtFramesAll, prFramesAll):
        if 'ignore_regions' in gtf.keys() and len(gtf['ignore_regions']) > 0:
            polys = [np.array([[p['x'][0], p['y'][0]] for p in region['point']], np.float64).reshape(-1, 2)
                     for region in gtf['ignore_regions']]
            for poly in polys:
                if len(poly) < 3:
                    raise ValueError('A LinearRing must have at least 3 coordinate tuples (ignore region with %d points)'
                                     % len(poly))
            prf['annorect'] = _remove_ignored_points_rects(prf['annorect'], polys)
            gtf['annorect'] = _remove_ignored_points_rects(gtf['annorect'], polys)
    return gtFramesAll, prFramesAll, filenames


# ---- flat arrays --------------------------------------------------------------------------------------------------------

class PoseTrackPack(object):
    """The loaded frames as flat arrays.  Frame f owns GT rows gt_off[f]:gt_off[f+1] and prediction rows
    pr_off[f]:pr_off[f+1].  gt_rect [NG, 4] head box, gt_kp [NG, 15, 3] (x, y, present), gt_tid [NG]; pr_kp [NP, 15, 4]
    (x, y, score, present), pr_tid [NP]; all coordinates and scores fp64 as the JSON holds them.  seq_id [F] is the GT
    file index; pair_off [F + 1] prefix-sums predictions x GT per frame (where the device keeps each frame's distances)."""

    def __init__(self, gtFramesAll, prFramesAll, seq_names=()):
        assert len(gtFramesAll) == len(prFramesAll)
        F = len(gtFramesAll)
        self.nframes = F
        self.seq_names = list(seq_names)
        self.seq_id = np.array([f['seq_id'] for f in gtFramesAll], np.int64)
        ng = np.array([len(f['annorect']) for f in gtFramesAll], np.int64)
        npr = np.array([len(f['annorect']) for f in prFramesAll], np.int64)
        self.gt_off = np.concatenate([[0], np.cumsum(ng)]).astype(np.int64)
        self.pr_off = np.concatenate([[0], np.cumsum(npr)]).astype(np.int64)
        self.pair_off = np.concatenate([[0], np.cumsum(ng * npr)]).astype(np.int64)
        NG, NP = int(self.gt_off[-1]), int(self.pr_off[-1])
        self.gt_rect = np.full((NG, 4), np.nan)
        self.gt_kp = np.zeros((NG, N_JOINTS, 3))
        self.gt_tid = np.full(NG, -1, np.int64)
        self.pr_kp = np.zeros((NP, N_JOINTS, 4))
        self.pr_tid = np.full(NP, -1, np.int64)
        self.all_tracked = True
        g = p = 0
        for gtf, prf in zip(gtFramesAll, prFramesAll):
            for rect in gtf['annorect']:
                for k, key in enumerate(('x1', 'y1', 'x2', 'y2')):
                    if key in rect.keys():
                        self.gt_rect[g, k] = rect[key][0]
                self.gt_tid[g] = self._track(rect)
                for i, pt in self._joints(rect).items():
                    self.gt_kp[g, i] = (pt['x'][0], pt['y'][0], 1.0)
                g += 1
            for rect in prf['annorect']:
                self.pr_tid[p] = self._track(rect)
                for i, pt in self._joints(rect).items():
                    if 'score' not in pt.keys():
                        raise ValueError('keypoint score is missing (prediction frame %s)' % prf.get('image', '?'))
                    self.pr_kp[p, i] = (pt['x'][0], pt['y'][0], pt['score'][0], 1.0)
                p += 1
        self.n_gt, self.n_pr = ng, npr
        self.max_gt = int(ng.max()) if F else 0
        self.max_pr = int(npr.max()) if F else 0
        self.has_mot = (ng > 0) & (npr > 0)

    def _track(self, rect):
        if 'track_id' in rect.keys():
            return int(rect['track_id'][0])
        self.all_tracked = False
        return -1

    @staticmethod
    def _joints(rect):
        """getPointGTbyID for every joint: the first point of each id."""
        out = {}
        if len(rect['annopoints']) > 0:
            for pt in rect['annopoints'][0]['point']:
                if pt['id'] is not None:
                    i = pt['id'][0]
                    if 0 <= i < N_JOINTS and i not in out:
                        out[i] = pt
        return out

    def validate(self):
        """The device limits, checked before any device call."""
        for f in range(self.nframes):
            if self.n_gt[f] > L.PT_MAX_GT:
                raise ValueError('frame %d has %d GT people (at most %d)' % (f, self.n_gt[f], L.PT_MAX_GT))
            if self.n_pr[f] > L.LSA_MAX_DIM:
                raise ValueError('frame %d has %d predicted people (at most %d)' % (f, self.n_pr[f], L.LSA_MAX_DIM))
        if self.pr_off[-1] * N_JOINTS >= 2 ** 30:
            raise ValueError('%d predictions x %d joints: more than 2^30 scores' % (self.pr_off[-1], N_JOINTS))

    def seq_ranges(self):
        """[(seq index, first frame, end frame)] of the sequences that kept frames, in order."""
        out = []
        if self.nframes:
            starts = np.flatnonzero(np.r_[True, self.seq_id[1:] != self.seq_id[:-1]])
            ends = np.r_[starts[1:], self.nframes]
            out = [(int(self.seq_id[a]), int(a), int(b)) for a, b in zip(starts, ends)]
        return out

    def frame_name(self, f):
        s = int(self.seq_id[f])
        name = osp.basename(self.seq_names[s]) if s < len(self.seq_names) else 'sequence %d' % s
        return 'frame %d (%s, frame %d of the sequence after cleanup)' % (f, name, f - int(np.searchsorted(self.seq_id, s)))


def mot_sources(pack, lo=0, hi=None):
    """The frame whose MOT inputs frame f uses, for f in [lo, hi): f itself when it has both GT and predictions, else
    the latest such frame before it in [lo, f) (the reference's stale ``mot``), -1 where there is none."""
    hi = pack.nframes if hi is None else hi
    idx = np.where(pack.has_mot[lo:hi], np.arange(lo, hi), -1)
    return np.maximum.accumulate(idx) if len(idx) else idx


# ---- host arithmetic of the reference on the per-joint sums -----------------------------------------------------------

def ap_metrics(seg_out):
    """evaluateAP.computeMetrics from the 15 per-joint (AP, precision, recall) x 100 -> apAll, preAll, recAll [16, 1]."""
    apAll, preAll, recAll = (np.zeros((N_JOINTS + 1, 1)) for _ in range(3))
    seg_out = np.asarray(seg_out, np.float64).reshape(N_JOINTS, 3)
    apAll[:N_JOINTS, 0], preAll[:N_JOINTS, 0], recAll[:N_JOINTS, 0] = seg_out[:, 0], seg_out[:, 1], seg_out[:, 2]
    apAll[N_JOINTS] = apAll[:N_JOINTS, 0].mean()
    recAll[N_JOINTS] = recAll[:N_JOINTS, 0].mean()
    preAll[N_JOINTS] = preAll[:N_JOINTS, 0].mean()
    return apAll, preAll, recAll


def mot_metrics(counts, sumd):
    """evaluateTracking.computeMetrics (:108-133) from the per-sequence event counts [S, 15, 4] (MATCH, SWITCH, FP,
    MISS) and distance sums [S, 15], summed over the sequences in order -> the metrics column [19, 1]."""
    counts = np.asarray(counts, np.int64).reshape(-1, N_JOINTS, 4)
    mid = {k: np.zeros([1, N_JOINTS]) for k in ('num_misses', 'num_switches', 'num_false_positives', 'num_objects',
                                                'num_detections', 'sumD')}
    for s in range(counts.shape[0]):
        m, sw, fp, miss = (counts[s, :, k] for k in range(4))
        mid['num_misses'][0] += miss
        mid['num_switches'][0] += sw
        mid['num_false_positives'][0] += fp
        mid['num_objects'][0] += m + sw + miss
        mid['num_detections'][0] += m + sw
        mid['sumD'][0] += np.asarray(sumd, np.float64).reshape(-1, N_JOINTS)[s]
    fin = {k: np.zeros([1, N_JOINTS + 1]) for k in ('mota', 'motp', 'pre', 'rec')}
    with np.errstate(divide='ignore', invalid='ignore'):
        for i in range(N_JOINTS):
            fin['mota'][0, i] = 100 * (1. - (mid['num_misses'][0, i] + mid['num_switches'][0, i] +
                                             mid['num_false_positives'][0, i]) / mid['num_objects'][0, i])
            numDet = mid['num_detections'][0, i]
            s = mid['sumD'][0, i]
            fin['motp'][0, i] = 0.0 if (numDet == 0 or np.isnan(s)) else 100 * (1. - (s / numDet))
            fin['pre'][0, i] = 100 * (mid['num_detections'][0, i] / (mid['num_detections'][0, i] +
                                                                      mid['num_false_positives'][0, i]))
            fin['rec'][0, i] = 100 * (mid['num_detections'][0, i] / mid['num_objects'][0, i])
        for k in fin:
            fin[k][0, N_JOINTS] = fin[k][0, :N_JOINTS].mean()
    metrics = np.full((N_JOINTS + 4, 1), np.nan)
    metrics[:N_JOINTS + 1, 0] = fin['mota'][0]
    metrics[N_JOINTS + 1, 0] = fin['motp'][0, N_JOINTS]
    metrics[N_JOINTS + 2, 0] = fin['pre'][0, N_JOINTS]
    metrics[N_JOINTS + 3, 0] = fin['rec'][0, N_JOINTS]
    return metrics


# ---- the device evaluation ----------------------------------------------------------------------------------------------

def _ap_segments(pack, groups):
    """One segment per (frame group, joint): (joint, first frame, end frame) and the score counts' prefix sums."""
    has = np.concatenate([np.zeros((1, N_JOINTS), np.int64), np.cumsum(pack.pr_kp[:, :, 3] != 0, axis=0)])
    segs, sizes = [], []
    for lo, hi in groups:
        for j in range(N_JOINTS):
            segs.append((j, lo, hi))
            sizes.append(int(has[pack.pr_off[hi], j] - has[pack.pr_off[lo], j]))
    return np.array(segs, np.int32).reshape(-1, 3), np.concatenate([[0], np.cumsum(sizes, dtype=np.int64)])


def _map_capacity(pack, lists):
    cap = 1
    for frames in lists:
        if len(frames):
            ids = np.concatenate([pack.gt_tid[pack.gt_off[f]:pack.gt_off[f + 1]] for f in np.unique(frames)])
            cap = max(cap, len(np.unique(ids)))
    if cap > L.PT_MAX_MAP_IDS:
        raise ValueError('a sequence sees %d distinct GT track ids (at most %d)' % (cap, L.PT_MAX_MAP_IDS))
    return cap


def evaluate_pack(pack, eval_pose=True, eval_track=True, per_video=False, track_upper_bound=False):
    """The device evaluation of a loaded pack.  With track_upper_bound, the MOT counts (total and per video) come from
    poseval's upper-bound view (assignGTmulti(..., computeUpperBound=True)): in every frame with both GT and predictions
    only the predictions some GT selected are kept, with that GT's track id; AP is unchanged.  Returns {'ap': (apAll, preAll, recAll), 'metrics': metrics} and, with
    per_video, 'videos': {seq index: (ap, mota)} as evaluating each GT file alone gives them (NaN where that fails).
    'raw' holds the device outputs: labels [NP, 15], ngt [15, F], the segments' (AP, precision, recall) [nseg, 3] (the
    15 joints of all frames first when eval_pose, then 15 per sequence with per_video), and the MOT counts [L, 15, 4] /
    sumd [L, 15] of the frame lists named by 'lists' (('all' | 'video' | 'failed', sequence); 'failed' has no row)."""
    pack.validate()
    nan16, nan19 = np.full((N_JOINTS + 1, 1), np.nan), np.full((N_JOINTS + 4, 1), np.nan)
    res = {'ap': (nan16, nan16.copy(), nan16.copy()), 'metrics': nan19, 'videos': {}}
    seqs = pack.seq_ranges()
    if eval_track:
        if not pack.all_tracked:
            raise ValueError('tracking evaluation needs a track_id in every GT and prediction rect')
        src = mot_sources(pack)
        if pack.nframes and (src < 0).any():
            raise ValueError('%s has no MOT inputs: neither it nor an earlier frame has both GT and predictions'
                             % pack.frame_name(int(np.flatnonzero(src < 0)[0])))
    if pack.nframes == 0 or not (eval_pose or eval_track or per_video):
        return res
    from ..ops import poseval_ops as P
    torch = L.require_cuda()
    dp = P.DevicePack(pack)
    labels, ngt, dist = P.assign(dp)
    groups = [(0, pack.nframes)] + ([(a, b) for _, a, b in seqs] if per_video else [])
    ap_out = None
    if eval_pose or per_video:
        segs, seg_off = _ap_segments(pack, groups if eval_pose else groups[1:])
        ap_out = P.average_precision(dp, labels, ngt, segs, seg_off)
    lists, kinds = [], []
    if eval_track:
        for s, a, b in seqs:                                  # process_frame drops each sequence's last frame
            lists.append(src[a:b - 1]); kinds.append(('all', s))
        if per_video:
            for s, a, b in seqs:
                vsrc = mot_sources(pack, a, b)
                if (vsrc < 0).any():
                    kinds.append(('failed', s))
                    continue
                lists.append(vsrc[:-1]); kinds.append(('video', s))
    mot_out = None
    if lists:
        list_off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
        frames = np.concatenate(lists).astype(np.int64)
        mdp = P.upper_bound(dp, dist) if track_upper_bound else dp
        counts, sumd, status = P.mot_counts(mdp, mdp.dist if track_upper_bound else dist, list_off, frames,
                                            _map_capacity(pack, lists))
        torch.cuda.synchronize()
        if int(status.max()) != 0:
            raise RuntimeError('dt_posetrack_mot: a frame list exceeded its bounds')
        mot_out = (counts.cpu().numpy(), sumd.cpu().numpy())
    ap_np = ap_out.cpu().numpy() if ap_out is not None else None
    res['raw'] = dict(labels=labels.cpu().numpy()[:int(pack.pr_off[-1])], ngt=ngt.cpu().numpy(), ap=ap_np,
                      counts=mot_out[0] if mot_out else None, sumd=mot_out[1] if mot_out else None, lists=kinds)
    if eval_pose:
        res['ap'] = ap_metrics(ap_np[:N_JOINTS])
    if eval_track:
        n_all = len(seqs)
        res['metrics'] = mot_metrics(mot_out[0][:n_all], mot_out[1][:n_all])
    if per_video:
        videos = {}
        base = N_JOINTS if eval_pose else 0
        li = len(seqs)
        for k, (s, a, b) in enumerate(seqs):
            ap = ap_metrics(ap_np[base + k * N_JOINTS:base + (k + 1) * N_JOINTS])[0][-1][0]
            mota = np.nan
            if eval_track:
                kind = [kd for kd in kinds if kd[1] == s and kd[0] != 'all'][0][0]
                if kind == 'failed':
                    ap = np.nan
                else:
                    mota = mot_metrics(mot_out[0][li:li + 1], mot_out[1][li:li + 1])[-4][0]
                    li += 1
            videos[s] = (ap, mota)
        res['videos'] = videos
    return res


# ---- printing (eval_helpers.printTable) ---------------------------------------------------------------------------------

def _format_cell(val, delim):
    return '{:>5}'.format('%1.1f' % val) + delim


def get_header():
    return '&' + ' Head &' + ' Shou &' + ' Elb  &' + ' Wri  &' + ' Hip  &' + ' Knee &' + ' Ankl &' + ' Total%s' % ('\\' + '\\')


def get_mot_header():
    h = '&' + ' MOTA &' * 8 + ' MOTP &' + ' Prec &' + ' Rec  %s\n' % ('\\' + '\\')
    h += '&' + ' Head &' + ' Shou &' + ' Elb  &' + ' Wri  &' + ' Hip  &' + ' Knee &' + ' Ankl &' + ' Total&' * 3
    return h + ' Total%s' % ('\\' + '\\')


def get_cum(vals):
    cum = [vals[[HEAD_TOP, NECK, NOSE], 0].mean(), vals[[RIGHT_SHOULDER, LEFT_SHOULDER], 0].mean(),
           vals[[RIGHT_ELBOW, LEFT_ELBOW], 0].mean(), vals[[RIGHT_WRIST, LEFT_WRIST], 0].mean(),
           vals[[RIGHT_HIP, LEFT_HIP], 0].mean(), vals[[RIGHT_KNEE, LEFT_KNEE], 0].mean(),
           vals[[RIGHT_ANKLE, LEFT_ANKLE], 0].mean()]
    return cum + [vals[i, 0] for i in range(N_JOINTS, len(vals))]


def get_format_row(cum):
    row = '&'
    for c in cum[:-1]:
        row += _format_cell(c, ' &')
    return row + _format_cell(cum[-1], (' %s' % '\\' + '\\'))


def print_table(vals, motHeader=False):
    """eval_helpers.printTable: prints and returns (header + newline, row + newline)."""
    row = get_format_row(get_cum(vals))
    header = get_mot_header() if motHeader else get_header()
    print(header)
    print(row)
    return header + '\n', row + '\n'



def evaluate(gtdir, preddir, eval_pose=True, eval_track=True, eval_upper_bound=False, per_video=False, verbose=True):
    """evaluate_simple.evaluate.  ((apAll, preAll, recAll) [16, 1], metrics [19, 1]), NaN where not evaluated; with
    per_video also {GT file name: (ap, mota)} as a third element.

    eval_upper_bound raises NotImplementedError: the upper bound replaces the predictions' track ids with the GT's, so a
    call that asks for it names it explicitly through evaluate_upper_bound(), and a MOTA from evaluate() is always the
    predictions' own."""
    if eval_upper_bound:
        raise NotImplementedError('evaluate() scores the predictions as they are; the upper-bound tracking evaluation '
                                  '(TRACKING.DEBUG.UPPER_BOUND_4_EVAL_UPPER_BOUND) is evaluate_upper_bound()')
    return _evaluate(gtdir, preddir, eval_pose, eval_track, False, per_video, verbose)


def evaluate_upper_bound(gtdir, preddir, eval_pose=True, eval_track=True, per_video=False, verbose=True):
    """evaluate_simple.evaluate(..., eval_upper_bound=True): as evaluate(), with the MOT metrics of poseval's upper bound
    (every prediction a GT selected takes that GT's track id, the others are dropped from the MOT inputs)."""
    return _evaluate(gtdir, preddir, eval_pose, eval_track, True, per_video, verbose)


def _evaluate(gtdir, preddir, eval_pose, eval_track, track_upper_bound, per_video, verbose):
    gtFramesAll, prFramesAll, names = load_data_dir(gtdir, preddir)
    if verbose:
        print('# gt frames  :', len(gtFramesAll))
        print('# pred frames:', len(prFramesAll))
    res = evaluate_pack(PoseTrackPack(gtFramesAll, prFramesAll, names), eval_pose, eval_track, per_video, track_upper_bound)
    if verbose and eval_pose:
        print('Average Precision (AP) metric:')
        print_table(res['ap'][0])
    if verbose and eval_track:
        print('Multiple Object Tracking (MOT) metrics:')
        print_table(res['metrics'], motHeader=True)
    out = (res['ap'], res['metrics'])
    if per_video:
        # a file whose frames all went in cleanup scores AP 0 and MOTA NaN on its own (0/0 objects)
        out += ({osp.basename(n): res['videos'].get(s, (0.0, np.nan)) for s, n in enumerate(names)},)
    return out
