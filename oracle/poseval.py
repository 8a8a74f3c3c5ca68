"""Oracle: the PoseTrack evaluation (TEST INFRASTRUCTURE ONLY, see oracle/__init__).

A py3 numpy restatement of the reference's vendored poseval (lib/datasets/posetrack/poseval/py/) as
``evaluate_simple.evaluate`` runs it:
  - load_data_dir + cleanupData + removeIgnoredPoints (eval_helpers.py:282-415), GT files in sorted order, ignore
    regions by exact rational point-in-polygon (shapely's Polygon.contains: the boundary is outside);
  - assignGTmulti (:423-637), with the stale ``motAll`` carry of its ``if 'mot' in locals()``;
  - computeRPC / VOCap (:169-207) and evaluateAP.computeMetrics, ties ranked by (score descending, position in the
    concatenation order); the reference's np.argsort leaves them to numpy's unstable sort;
  - py-motmetrics' MOTAccumulator.update (motmetrics/mot.py:90-191) with scipy.optimize.linear_sum_assignment, and
    evaluateTracking.computeMetrics over the per-sequence event counts (motmetrics/metrics.py definitions).
Distances are sqrt(dx*dx + dy*dy) in Python floats (no fused multiply-add), as the device computes them.
"""
import glob
import json
import math
import os.path as osp
from fractions import Fraction

import numpy as np
from scipy.optimize import linear_sum_assignment

N_JOINTS = 15
MAX_TRACK_ID = 1000


# ---- loader -------------------------------------------------------------------------------------------------------------

def polygon_contains(poly, x, y):
    """Exact: (x, y) strictly inside the polygon (even-odd rule), on an edge or vertex is outside."""
    if len(poly) < 3:
        raise ValueError('A LinearRing must have at least 3 coordinate tuples')
    P = [(Fraction(a), Fraction(b)) for a, b in poly]
    px, py = Fraction(x), Fraction(y)
    inside = False
    for k in range(len(P)):
        (ax, ay), (bx, by) = P[k], P[(k + 1) % len(P)]
        o = (ax - px) * (by - py) - (ay - py) * (bx - px)
        if o == 0 and min(ax, bx) <= px <= max(ax, bx) and min(ay, by) <= py <= max(ay, by):
            return False
        if (ay > py) != (by > py) and ((o > 0) if by > ay else (o < 0)):
            inside = not inside
    return inside


def _has_points(rect):
    return (('annopoints' in rect.keys()) and (len(rect['annopoints']) > 0 and len(rect['annopoints'][0]) > 0) and
            ('point' in rect['annopoints'][0].keys()))


def load_data_dir(gt_dir, pred_dir):
    filenames = sorted(glob.glob(osp.join(gt_dir, '*.json')))
    gtAll, prAll = [], []
    for i, fname in enumerate(filenames):
        gt = json.load(open(fname))['annolist']
        for frame in gt:
            frame['seq_id'] = i
            for rect in frame['annorect']:
                if 'track_id' in rect.keys():
                    assert rect['track_id'][0] < MAX_TRACK_ID
                    rect['track_id'][0] += i * MAX_TRACK_ID
        gtAll += gt
        pname = osp.join(pred_dir, osp.basename(fname))
        if not osp.exists(pname):
            raise IOError('Prediction file ' + pname + ' does not exist')
        pr = json.load(open(pname))['annolist']
        if len(pr) != len(gt):
            raise Exception('# prediction frames %d <> # GT frames %d for %s' % (len(pr), len(gt), pname))
        for frame in pr:
            for rect in frame['annorect']:
                if 'track_id' in rect.keys():
                    assert rect['track_id'][0] < MAX_TRACK_ID
                    rect['track_id'][0] += i * MAX_TRACK_ID
        prAll += pr
    keep = [k for k in range(len(gtAll)) if len(gtAll[k]['annorect']) > 0]
    gtAll, prAll = [gtAll[k] for k in keep], [prAll[k] for k in keep]
    for g, p in zip(gtAll, prAll):
        g['annorect'] = [r for r in g['annorect'] if _has_points(r)]
        p['annorect'] = [r for r in p['annorect'] if _has_points(r)]
    for g, p in zip(gtAll, prAll):
        if 'ignore_regions' in g.keys() and len(g['ignore_regions']) > 0:
            polys = [[(q['x'][0], q['y'][0]) for q in reg['point']] for reg in g['ignore_regions']]
            for poly in polys:
                if len(poly) < 3:
                    raise ValueError('A LinearRing must have at least 3 coordinate tuples')
            for fr in (p, g):
                rects = []
                for rect in fr['annorect']:
                    pts = [q for q in rect['annopoints'][0]['point']
                           if not any(polygon_contains(poly, q['x'][0], q['y'][0]) for poly in polys)]
                    if pts:
                        rect['annopoints'][0]['point'] = pts
                        rects.append(rect)
                fr['annorect'] = rects
    return gtAll, prAll, filenames


# ---- assignGTmulti ------------------------------------------------------------------------------------------------------

def _point(points, i):
    for q in points:
        if q['id'] is not None and q['id'][0] == i:
            return q
    return None


def assign_gt_multi(gtFrames, prFrames, distThresh=0.5):
    """-> scoresAll[j][f], labelsAll[j][f] (lists), nGTall [15, F], motAll {f: {j: {...}}} (stale frames share inputs)."""
    F = len(gtFrames)
    scoresAll = [[[] for _ in range(F)] for _ in range(N_JOINTS)]
    labelsAll = [[[] for _ in range(F)] for _ in range(N_JOINTS)]
    nGTall = np.zeros([N_JOINTS, F])
    motAll, mot = {}, None
    for f in range(F):
        gts, prs = gtFrames[f]['annorect'], prFrames[f]['annorect']
        nG, nP = len(gts), len(prs)
        hasGT = np.zeros((nG, N_JOINTS), bool)
        gxy = np.zeros((nG, N_JOINTS, 2))
        tG = [r['track_id'][0] if 'track_id' in r.keys() else -1 for r in gts]
        for g, r in enumerate(gts):
            pts = r['annopoints'][0]['point'] if len(r['annopoints']) > 0 else []
            for i in range(N_JOINTS):
                q = _point(pts, i)
                if q is not None:
                    hasGT[g, i] = True
                    gxy[g, i] = (q['x'][0], q['y'][0])
        hasPr = np.zeros((nP, N_JOINTS), bool)
        score = np.full((nP, N_JOINTS), np.nan)
        pxy = np.zeros((nP, N_JOINTS, 2))
        tP = [r['track_id'][0] if 'track_id' in r.keys() else -1 for r in prs]
        for p, r in enumerate(prs):
            for i in range(N_JOINTS):
                q = _point(r['annopoints'][0]['point'], i)
                if q is not None:
                    hasPr[p, i] = True
                    score[p, i] = q['score'][0]
                    pxy[p, i] = (q['x'][0], q['y'][0])
        if nP and nG:
            dist = np.full((nP, nG, N_JOINTS), np.inf)
            for g, r in enumerate(gts):
                head = 0.6 * math.sqrt((r['x2'][0] - r['x1'][0]) * (r['x2'][0] - r['x1'][0]) +
                                       (r['y2'][0] - r['y1'][0]) * (r['y2'][0] - r['y1'][0]))
                dx = gxy[g, :, 0][None, :] - pxy[:, :, 0]
                dy = gxy[g, :, 1][None, :] - pxy[:, :, 1]
                with np.errstate(divide='ignore', invalid='ignore'):
                    d = np.sqrt(dx * dx + dy * dy) / head
                both = hasPr & hasGT[g][None, :]
                dist[:, g, :] = np.where(both, d, np.inf)
            nGTp = hasGT.sum(axis=1)
            match = dist <= distThresh
            pck = 1.0 * match.sum(axis=2)
            for j in range(nG):
                if nGTp[j] > 0:
                    pck[:, j] = pck[:, j] / nGTp[j]
            idx = np.argmax(pck, axis=1)
            for p in range(nP):
                keep = pck[p, idx[p]]
                pck[p, :] = 0
                pck[p, idx[p]] = keep
            prToGT = np.argmax(pck, axis=0)
            prToGT[np.max(pck, axis=0) == 0] = -1
            mot = {}
            for i in range(N_JOINTS):
                rg = np.flatnonzero(hasGT[:, i])
                rp = np.flatnonzero(hasPr[:, i])
                dd = np.full((len(rg), len(rp)), np.nan)
                for a, g in enumerate(rg):
                    for b, p in enumerate(rp):
                        if match[p, g, i]:
                            dd[a, b] = dist[p, g, i]
                mot[i] = {'trackidxGT': [tG[g] for g in rg], 'trackidxPr': [tP[p] for p in rp], 'dist': dd}
            for p in range(nP):
                hit = np.flatnonzero(prToGT == p)
                for i in range(N_JOINTS):
                    if hasPr[p, i]:
                        scoresAll[i][f].append(score[p, i])
                        labelsAll[i][f].append(int(match[p, hit[0], i]) if len(hit) else 0)
        elif not nG:
            for p in range(nP):
                for i in range(N_JOINTS):
                    if hasPr[p, i]:
                        scoresAll[i][f].append(score[p, i])
                        labelsAll[i][f].append(0)
        nGTall[:, f] += hasGT.sum(axis=0)
        if mot is not None:
            motAll[f] = mot
    return scoresAll, labelsAll, nGTall, motAll


# ---- AP -----------------------------------------------------------------------------------------------------------------

def sort_order(scores):
    """Score descending (NaN first, as argsort()[::-1] puts it), ties by position."""
    s = np.asarray(scores, np.float64)
    return np.lexsort((np.arange(len(s)), -np.where(np.isnan(s), 0, s), ~np.isnan(s)))


def compute_rpc(scores, labels, totalPos):
    order = sort_order(scores)
    labels = np.asarray(labels)[order]
    precision, recall = np.zeros(len(order)), np.zeros(len(order))
    npos = 0
    with np.errstate(divide='ignore', invalid='ignore'):
        for k in range(len(order)):
            if labels[k] == 1:
                npos += 1
            recall[k] = 1.0 * npos / np.float64(totalPos)
            precision[k] = 1.0 * npos / (k + 1)
    return precision, recall, order


def voc_ap(rec, prec):
    mpre = np.zeros([1, 2 + len(prec)])
    mpre[0, 1:len(prec) + 1] = prec
    mrec = np.zeros([1, 2 + len(rec)])
    mrec[0, 1:len(rec) + 1] = rec
    mrec[0, len(rec) + 1] = 1.0
    for i in range(mpre.size - 2, -1, -1):
        mpre[0, i] = max(mpre[0, i], mpre[0, i + 1])
    i = (np.argwhere(~np.equal(mrec[0, 1:], mrec[0, :mrec.shape[1] - 1])) + 1).flatten()
    with np.errstate(invalid='ignore'):
        return np.sum(np.multiply(np.subtract(mrec[0, i], mrec[0, i - 1]), mpre[0, i]))


def ap_metrics(scoresAll, labelsAll, nGTall, frames=None):
    """evaluateAP.computeMetrics over the frames (all by default) -> apAll, preAll, recAll [16, 1]."""
    frames = range(nGTall.shape[1]) if frames is None else frames
    apAll, preAll, recAll = (np.zeros((N_JOINTS + 1, 1)) for _ in range(3))
    for j in range(N_JOINTS):
        scores = [s for f in frames for s in scoresAll[j][f]]
        labels = [l for f in frames for l in labelsAll[j][f]]
        nGT = sum(nGTall[j, list(frames)])
        precision, recall, _ = compute_rpc(scores, labels, nGT)
        if len(precision) > 0:
            apAll[j] = voc_ap(recall, precision) * 100
            preAll[j] = precision[-1] * 100
            recAll[j] = recall[-1] * 100
    apAll[N_JOINTS] = apAll[:N_JOINTS, 0].mean()
    recAll[N_JOINTS] = recAll[:N_JOINTS, 0].mean()
    preAll[N_JOINTS] = preAll[:N_JOINTS, 0].mean()
    return apAll, preAll, recAll


# ---- CLEAR MOT ----------------------------------------------------------------------------------------------------------

class MOTAccumulator(object):
    """MOTAccumulator(auto_id=True) with an event list instead of the pandas frame; max_switch_time is infinite."""

    def __init__(self):
        self.m = {}
        self.events = []          # (type, oid, hid, d)

    def update(self, oids, hids, dists):
        oids = np.ma.array(oids, mask=np.zeros(len(oids)))
        hids = np.ma.array(hids, mask=np.zeros(len(hids)))
        dists = np.atleast_2d(dists).astype(float).reshape(oids.shape[0], hids.shape[0]).copy()
        valid = dists[np.isfinite(dists)]
        INVDIST = 2 * valid.max() + 1 if valid.shape[0] > 0 else 1.
        dists[~np.isfinite(dists)] = INVDIST
        if oids.size * hids.size > 0:
            for i in range(oids.shape[0]):
                if not oids[i] in self.m:
                    continue
                hprev = self.m[oids[i]]
                j, = np.where(hids == hprev)
                if j.shape[0] == 0:
                    continue
                j = j[0]
                if not dists[i, j] == INVDIST:
                    oids[i] = np.ma.masked
                    hids[j] = np.ma.masked
                    self.m[oids.data[i]] = hids.data[j]
                    self.events.append(('MATCH', oids.data[i], hids.data[j], dists[i, j]))
            dists[oids.mask, :] = INVDIST
            dists[:, hids.mask] = INVDIST
            rids, cids = linear_sum_assignment(dists)
            for i, j in zip(rids, cids):
                if dists[i, j] == INVDIST:
                    continue
                o = oids[i]
                h = hids.data[j]
                cat = 'SWITCH' if (o in self.m and self.m[o] != h) else 'MATCH'
                self.events.append((cat, oids.data[i], hids.data[j], dists[i, j]))
                oids[i] = np.ma.masked
                hids[j] = np.ma.masked
                self.m[o] = h
        for o in oids[~oids.mask]:
            self.events.append(('MISS', o, np.nan, np.nan))
        for h in hids[~hids.mask]:
            self.events.append(('FP', np.nan, h, np.nan))

    def counts(self):
        """(MATCH, SWITCH, FP, MISS) and the distance sum (metrics.py: num_matches ... / df['D'].sum())."""
        c = [sum(1 for e in self.events if e[0] == t) for t in ('MATCH', 'SWITCH', 'FP', 'MISS')]
        d = np.array([e[3] for e in self.events if e[0] in ('MATCH', 'SWITCH')], np.float64)
        return c, float(np.sum(d)) if len(d) else 0.0


def mot_sequence_counts(seq_frames, motAll):
    """process_frame for one sequence's frame indices -> counts [15, 4], sumd [15]; KeyError where a frame has no
    MOT inputs, as the reference."""
    counts, sumd = np.zeros((N_JOINTS, 4), np.int64), np.zeros(N_JOINTS)
    for i in range(N_JOINTS):
        acc = MOTAccumulator()
        for f in seq_frames[:-1]:
            acc.update(motAll[f][i]['trackidxGT'], motAll[f][i]['trackidxPr'], motAll[f][i]['dist'])
        counts[i], sumd[i] = acc.counts()
    return counts, sumd


def mot_metrics(counts, sumd):
    """evaluateTracking.computeMetrics from the per-sequence counts [S, 15, 4] and sums [S, 15] -> metrics [19, 1]."""
    mid = {k: np.zeros([1, N_JOINTS]) for k in ('miss', 'sw', 'fp', 'obj', 'det', 'sumD')}
    for s in range(len(counts)):
        m, sw, fp, miss = (np.asarray(counts[s])[:, k] for k in range(4))
        mid['miss'][0] += miss
        mid['sw'][0] += sw
        mid['fp'][0] += fp
        mid['obj'][0] += m + sw + miss
        mid['det'][0] += m + sw
        mid['sumD'][0] += sumd[s]
    fin = {k: np.zeros([1, N_JOINTS + 1]) for k in ('mota', 'motp', 'pre', 'rec')}
    with np.errstate(divide='ignore', invalid='ignore'):
        for i in range(N_JOINTS):
            fin['mota'][0, i] = 100 * (1. - (mid['miss'][0, i] + mid['sw'][0, i] + mid['fp'][0, i]) / mid['obj'][0, i])
            numDet, s = mid['det'][0, i], mid['sumD'][0, i]
            fin['motp'][0, i] = 0.0 if (numDet == 0 or np.isnan(s)) else 100 * (1. - (s / numDet))
            fin['pre'][0, i] = 100 * (mid['det'][0, i] / (mid['det'][0, i] + mid['fp'][0, i]))
            fin['rec'][0, i] = 100 * (mid['det'][0, i] / mid['obj'][0, i])
        for k in fin:
            fin[k][0, N_JOINTS] = fin[k][0, :N_JOINTS].mean()
    metrics = np.full((N_JOINTS + 4, 1), np.nan)
    metrics[:N_JOINTS + 1, 0] = fin['mota'][0]
    metrics[N_JOINTS + 1:, 0] = [fin['motp'][0, N_JOINTS], fin['pre'][0, N_JOINTS], fin['rec'][0, N_JOINTS]]
    return metrics


def sequences(gtFrames):
    seq = np.array([f['seq_id'] for f in gtFrames], np.int64)
    return [(int(s), np.flatnonzero(seq == s)) for s in np.unique(seq)]


def evaluate_frames(gtFrames, prFrames, eval_pose=True, eval_track=True):
    """evaluate_simple.evaluate on loaded frames -> ((apAll, preAll, recAll), metrics, per-sequence (counts, sumd))."""
    ap = tuple(np.full((N_JOINTS + 1, 1), np.nan) for _ in range(3))
    metrics = np.full((N_JOINTS + 4, 1), np.nan)
    scoresAll, labelsAll, nGTall, motAll = assign_gt_multi(gtFrames, prFrames)
    if eval_pose:
        ap = ap_metrics(scoresAll, labelsAll, nGTall)
    per_seq = None
    if eval_track:
        assert len(gtFrames) == len(motAll)
        per_seq = [mot_sequence_counts(frames, motAll) for _, frames in sequences(gtFrames)]
        metrics = mot_metrics([c for c, _ in per_seq], [d for _, d in per_seq])
    return ap, metrics, per_seq


def evaluate(gtdir, preddir, eval_pose=True, eval_track=True):
    gtFrames, prFrames, _ = load_data_dir(gtdir, preddir)
    ap, metrics, _ = evaluate_frames(gtFrames, prFrames, eval_pose, eval_track)
    return ap, metrics


def evaluate_per_video(gtdir, preddir, eval_track=True):
    """{GT file name: (total AP, total MOTA)} evaluating each file alone (mpii_eval_engine._run_eval_single_video),
    NaN for both where that fails."""
    gtFrames, prFrames, names = load_data_dir(gtdir, preddir)
    out = {}
    for s, name in enumerate(names):
        idx = [k for k, f in enumerate(gtFrames) if f['seq_id'] == s]
        g = [dict(gtFrames[k], seq_id=0) for k in idx]
        p = [prFrames[k] for k in idx]              # the file's track-id offset changes no count
        try:
            (apAll, _, _), metrics, _ = evaluate_frames(g, p, True, eval_track)
            out[osp.basename(name)] = (apAll[-1][0], metrics[-4][0])
        except (AssertionError, KeyError):
            out[osp.basename(name)] = (np.nan, np.nan)
    return out
