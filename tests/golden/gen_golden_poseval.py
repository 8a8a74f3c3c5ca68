"""Golden vectors for the PoseTrack evaluation, from the REFERENCE's own poseval source.

    python tests/golden/gen_golden_poseval.py     -> tests/golden/poseval.npz

What runs, from the reference's source text (lib/datasets/posetrack/poseval/py/, Python 2):
    eval_helpers.py: Joint (:8-59), getPointGTbyID / getHeadSize (:62-75), computeRPC / VOCap (:168-207), help /
    process_arguments (:213-235), cleanupData ... load_data_dir (:282-415), assignGTmulti (:423-637);
    evaluateAP.py: computeMetrics / evaluateAP (:9-45);
    evaluateTracking.py: process_frame / computeMetrics / evaluateTracking (:15-148);
    py-motmetrics mot.py: MOTAccumulator.update / _sanitize_dists (:90-191, :214-229) on an event-list storage;
    py-motmetrics metrics.py: num_matches ... num_objects (:196-218) on a pandas frame of those events.
Shims: ``<>`` reads ``!=``; ``glob.glob`` is sorted (the GT file order this project documents); shapely's
``geometry.Polygon.contains`` is an exact rational point-in-polygon test (the boundary is outside, fewer than 3 points
raise ValueError); ``mp.Pool`` maps in process; ``print`` is silent; the MOTAccumulator events live in a list whose
``auto_id`` frame id is the number of distinct frame ids so far.  computeRPC's ``np.array(scores).argsort()[::-1]``
(numpy's unstable sort) is replaced by the documented tie rule: score descending, then position.

Cases (each a GT and a prediction directory, stored as '<case>/files', the JSON text of {'gt': {file name: annolist},
'pred': {...}}; posetrack_synth.write_dirs() lays them out):
  edge      hand-made: several sequences, ignore regions with joints on an edge and a vertex, GT rects without points,
            GT frames emptied by cleanup, prediction frames without rects (stale MOT inputs, across a sequence boundary
            too), carried-forward pairs, switches, duplicate hypothesis ids, a joint never annotated (0/0), the writer's
            -100 dummy predictions, frames where INVDIST pairs decide the assignment;
  synth     posetrack_synth.make_videos(4 videos of 16 frames, up to 8 GT and 12 predictions, seed 2);
  val3      3 videos of PoseTrack v1.0 val (lib/datasets/lists/PoseTrack/v1.0/posetrack_val.json), their first 8
            labelled frames: real head boxes,
            track ids and keypoints mapped by joint name; predictions are jittered GT with dropped joints, false
            positives and swapped ids.
Arrays per case: apAll / preAll / recAll [16, 1], metrics [19, 1] (evaluate_simple's layout), seq_counts [S, 15, 4]
(MATCH, SWITCH, FP, MISS per sequence and joint), seq_sumd [S, 15], labels [N] with labels_off [16] (per joint, in the
concatenation order) and ngt [15, F]; loaded: the JSON text of load_data_dir's (gtFramesAll, prFramesAll).
"""
import copy
import glob as _glob
import json
import os
import sys
import tempfile
import types
from fractions import Fraction
from functools import partial
from itertools import count

import numpy as np
import numpy.ma as ma
from scipy.optimize import linear_sum_assignment

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
PY = '/root/reference/lib/datasets/posetrack/poseval/py/'
MM = '/root/reference/lib/datasets/posetrack/poseval/py-motmetrics/motmetrics/'
VAL = '/root/reference/lib/datasets/lists/PoseTrack/v1.0/posetrack_val.json'
J = 15


# ---- shims --------------------------------------------------------------------------------------------------------------

class _Point(object):
    def __init__(self, x, y):
        self.x, self.y = x, y


class _Polygon(object):
    def __init__(self, coords):
        if len(coords) < 3:
            raise ValueError('A LinearRing must have at least 3 coordinate tuples')
        self.P = [(Fraction(a), Fraction(b)) for a, b in coords]

    def contains(self, pt):
        px, py = Fraction(pt.x), Fraction(pt.y)
        inside = False
        for k in range(len(self.P)):
            (ax, ay), (bx, by) = self.P[k], self.P[(k + 1) % len(self.P)]
            o = (ax - px) * (by - py) - (ay - py) * (bx - px)
            if o == 0 and min(ax, bx) <= px <= max(ax, bx) and min(ay, by) <= py <= max(ay, by):
                return False
            if (ay > py) != (by > py) and ((o > 0) if by > ay else (o < 0)):
                inside = not inside
        return inside


def _stable_desc(scores):
    s = np.asarray(scores, np.float64)
    return np.lexsort((np.arange(len(s)), -np.where(np.isnan(s), 0, s), ~np.isnan(s)))


class _Events(object):
    """The part of the pandas event frame MOTAccumulator.update touches."""

    def __init__(self):
        self.keys, self.rows = [], []
        ev = self

        class _Loc(object):
            def __setitem__(self, key, val):
                ev.keys.append(key[0])
                ev.rows.append(list(val))

            def __getitem__(self, fid):
                return [r for k, r in zip(ev.keys, ev.rows) if k[0] == fid]

        class _Index(object):
            def get_level_values(self, level):
                seen = []
                for k in ev.keys:
                    if k[level] not in seen:
                        seen.append(k[level])
                return types.SimpleNamespace(unique=lambda: np.array(seen))

            def __contains__(self, fid):
                return any(k[0] == fid for k in ev.keys)

        self.loc, self.index = _Loc(), _Index()

    def __getitem__(self, col):
        d = np.array([r[3] for r in self.rows], np.float64)
        return types.SimpleNamespace(sum=lambda: float(np.sum(np.where(np.isnan(d), 0.0, d))))

    def frame(self):
        import pandas as pd
        return pd.DataFrame(self.rows, columns=['Type', 'OId', 'HId', 'D'])


def _source(path, ranges, replace=()):
    src = open(path).read().split('\n')
    text = '\n'.join('\n'.join(src[a - 1:b]) for a, b in ranges)
    for old, new in replace:
        assert old in text, old
        text = text.replace(old, new)
    return text


def _method_source(path, first, last):
    lines = open(path).read().split('\n')[first - 1:last]
    return '\n'.join(l[4:] if l.startswith('    ') else l for l in lines)


def reference():
    """The reference's evaluation functions, executed from its source."""
    helpers = {'np': np, 'os': os, 'json': json, 'sys': sys, 'print': lambda *a, **k: None,
               'glob': types.SimpleNamespace(glob=lambda p: sorted(_glob.glob(p))),
               'geometry': types.SimpleNamespace(Point=_Point, Polygon=_Polygon), '_stable_desc': _stable_desc}
    exec(_source(PY + 'eval_helpers.py', [(8, 75), (168, 207), (213, 235), (282, 415), (423, 637)],
                 replace=[('(len(pr) <> len(gt))', '(len(pr) != len(gt))'),
                          ('idxsSort = np.array(scores).argsort()[::-1]', 'idxsSort = _stable_desc(scores)')]), helpers)
    eh = types.SimpleNamespace(**helpers)
    # py-motmetrics: the accumulator's own update() on the event list, the metrics on a pandas frame of it
    acc_ns = {'np': np, 'ma': ma, 'count': count, 'linear_sum_assignment': linear_sum_assignment}
    exec(_method_source(MM + 'mot.py', 90, 191), acc_ns)
    exec(_method_source(MM + 'mot.py', 214, 229), acc_ns)

    class MOTAccumulator(object):
        update = acc_ns['update']
        _sanitize_dists = acc_ns['_sanitize_dists']

        def __init__(self, auto_id=False, max_switch_time=float('inf')):
            self.auto_id, self.max_switch_time = auto_id, max_switch_time
            self.events, self.m, self.last_occurrence = _Events(), {}, {}

    met = {}
    exec(_source(MM + 'metrics.py', [(196, 218)]), met)

    def compute(acc, metrics=None, return_dataframe=False, name=None):
        df = acc.events.frame()
        nm, ns = met['num_matches'](df), met['num_switches'](df)
        vals = {'num_misses': met['num_misses'](df), 'num_switches': ns, 'num_false_positives': met['num_false_positives'](df),
                'num_objects': met['num_objects'](df), 'num_detections': met['num_detections'](df, nm, ns), 'num_matches': nm}
        return {k: vals[k] for k in metrics}

    mm = types.SimpleNamespace(MOTAccumulator=MOTAccumulator, metrics=types.SimpleNamespace(
        create=lambda: types.SimpleNamespace(compute=compute)))
    mp = types.SimpleNamespace(Pool=lambda n: types.SimpleNamespace(map=lambda f, it: list(map(f, it))))
    ap_ns = {'np': np, 'eval_helpers': eh}
    exec(_source(PY + 'evaluateAP.py', [(9, 45)]), ap_ns)
    tr_ns = {'np': np, 'mm': mm, 'mp': mp, 'partial': partial, 'eval_helpers': eh, 'Joint': eh.Joint,
             'print': lambda *a, **k: None}
    exec(_source(PY + 'evaluateTracking.py', [(15, 148)]), tr_ns)
    return eh, ap_ns, tr_ns


def run_reference(gt_dir, pred_dir):
    eh, ap_ns, tr_ns = reference()
    gtFramesAll, prFramesAll = eh.load_data_dir(['', gt_dir, pred_dir])
    scoresAll, labelsAll, nGTall, motAll = eh.assignGTmulti(copy.deepcopy(gtFramesAll), copy.deepcopy(prFramesAll), 0.5)
    apAll, preAll, recAll = ap_ns['evaluateAP'](copy.deepcopy(gtFramesAll), copy.deepcopy(prFramesAll))
    metricsAll = tr_ns['evaluateTracking'](copy.deepcopy(gtFramesAll), copy.deepcopy(prFramesAll), False)
    metrics = np.full((J + 4, 1), np.nan)
    for i in range(J + 1):
        metrics[i, 0] = metricsAll['mota'][0, i]
    metrics[J + 1, 0] = metricsAll['motp'][0, J]
    metrics[J + 2, 0] = metricsAll['pre'][0, J]
    metrics[J + 3, 0] = metricsAll['rec'][0, J]
    # per-sequence events, through the reference's process_frame
    seqidxs = np.array([f['seq_id'] for f in gtFramesAll])
    uniq = np.unique(seqidxs)
    names = ['num_misses', 'num_switches', 'num_false_positives', 'num_objects', 'num_detections']
    counts, sumd = np.zeros((len(uniq), J, 4), np.int64), np.zeros((len(uniq), J))
    for si in range(len(uniq)):
        mids, accs = tr_ns['process_frame'](si, J, seqidxs, uniq, motAll, names)
        for i in range(J):
            df = accs[i].events.frame()
            counts[si, i] = [(df.Type == t).sum() for t in ('MATCH', 'SWITCH', 'FP', 'MISS')]
            assert counts[si, i, 3] == mids[i]['num_misses'] and counts[si, i, 1] == mids[i]['num_switches']
            sumd[si, i] = accs[i].events['D'].sum()
    labels = [np.concatenate([np.asarray(labelsAll[j][f], np.int64).ravel() for f in range(len(gtFramesAll))] or
                             [np.zeros(0, np.int64)]) for j in range(J)]
    return dict(loaded=np.array(json.dumps([gtFramesAll, prFramesAll])),
                apAll=apAll, preAll=preAll, recAll=recAll, metrics=metrics, seq_counts=counts, seq_sumd=sumd,
                labels=np.concatenate(labels), labels_off=np.concatenate([[0], np.cumsum([len(l) for l in labels])]),
                ngt=nGTall.astype(np.int64))


# ---- cases --------------------------------------------------------------------------------------------------------------

def _pt(j, x, y, s=None):
    p = {'id': [j], 'x': [float(x)], 'y': [float(y)]}
    if s is not None:
        p['score'] = [float(s)]
    return p


def _gt_rect(tid, cx, cy, head=20.0, joints=range(J), jitter=None):
    pts = [_pt(j, cx + 3.0 * (j % 5) - 6.0, cy + 4.0 * (j // 5) - 4.0) for j in joints]
    return {'x1': [cx - head / 2], 'y1': [cy - 40 - head / 2], 'x2': [cx + head / 2], 'y2': [cy - 40 + head / 2],
            'track_id': [tid], 'annopoints': [{'point': pts}]}


def _pr_rect(tid, cx, cy, scores, off=0.0, joints=range(J)):
    pts = [_pt(j, cx + 3.0 * (j % 5) - 6.0 + off, cy + 4.0 * (j // 5) - 4.0, scores[j]) for j in joints]
    return {'annopoints': [{'point': pts}], 'score': [0.9], 'track_id': [tid]}


DUMMY = {'annopoints': [{'point': [_pt(0, 0, 0, -100.0)]}], 'score': [0], 'track_id': [0]}


def edge_case():
    rng = np.random.RandomState(5)
    no7 = [j for j in range(J) if j != 7]                  # joint 7 is never annotated: its AP is 0/0
    videos = {}
    for v in range(3):
        gt, pr = [], []
        for f in range(9):
            sc = np.round(rng.rand(J), 2)
            g = [_gt_rect(1, 100, 100, joints=no7), _gt_rect(2, 200, 100, joints=no7), _gt_rect(3, 300, 100, joints=no7)]
            p = [_pr_rect(11, 100, 100, sc), _pr_rect(12, 200, 100, sc, off=4.0), _pr_rect(13, 300, 100, sc, off=15.0)]
            if f >= 4:                                         # a real switch: hypotheses 11 and 12 trade people
                p[0]['track_id'], p[1]['track_id'] = [12], [11]
            if f == 2:                                         # duplicate hypothesis ids
                p[2]['track_id'] = [11]
                p.append(_pr_rect(11, 100, 100, sc, off=1.0))
            if f == 3:                                         # INVDIST decides: only far pairs are left after step 1
                p = [_pr_rect(11, 100, 100, sc), _pr_rect(12, 100, 100, sc, off=30.0), _pr_rect(13, 300, 100, sc, off=2.0)]
            if f == 5:
                g[1] = {'track_id': [2], 'x1': [0], 'y1': [0], 'x2': [1], 'y2': [1]}          # a GT rect without points
            if f == 6:
                g = [dict(r, annopoints=[]) for r in g]           # every rect loses its points: no GT in the frame
            if f == 7:                                         # ignore regions: joints on a vertex and on an edge
                x0, y0 = g[0]['annopoints'][0]['point'][0]['x'][0], g[0]['annopoints'][0]['point'][0]['y'][0]
                xe = g[1]['annopoints'][0]['point'][1]['x'][0]
                ye = g[1]['annopoints'][0]['point'][1]['y'][0]
                regions = [{'point': [_pt(0, x0, y0), _pt(1, x0 + 9, y0), _pt(2, x0 + 9, y0 + 9), _pt(3, x0, y0 + 9)]},
                           {'point': [_pt(0, xe - 2, ye), _pt(1, xe + 5, ye), _pt(2, xe + 5, ye + 5), _pt(3, xe - 2, ye + 5)]},
                           {'point': [_pt(0, 280, 80), _pt(1, 320, 80), _pt(2, 320, 120), _pt(3, 280, 120)]}]
            if f == 1 and v == 1:
                p = []                                         # stale MOT inputs from the previous frame
            if f == 0 and v == 2:
                p = []                                         # stale MOT inputs across the sequence boundary
            if f == 8:
                p = [copy.deepcopy(DUMMY)]                      # the writer's dummy prediction
            frame_g = {'image': [{'name': 'images/v%d/%05d.jpg' % (v, f)}], 'annorect': g}
            if f == 7:
                frame_g['ignore_regions'] = regions
            if f == 4 and v == 0:
                frame_g['annorect'] = []                       # removed by cleanupData, with its prediction frame
            gt.append(frame_g)
            pr.append({'image': 'images/v%d/%05d.jpg' % (v, f), 'annorect': p + ([copy.deepcopy(DUMMY)] if f == 2 else [])})
        videos['v%d.json' % v] = ({'annolist': gt}, {'annolist': pr})
    return videos


# PoseTrack 17-name order of posetrack_val.json -> the 15 joints of eval_helpers.Joint ('neck' is 'head_bottom')
_VAL_NAMES = ['nose', 'head_bottom', 'head_top', 'left_ear', 'right_ear', 'left_shoulder', 'right_shoulder', 'left_elbow',
              'right_elbow', 'left_wrist', 'right_wrist', 'left_hip', 'right_hip', 'left_knee', 'right_knee', 'left_ankle',
              'right_ankle']
_DST = ['right_ankle', 'right_knee', 'right_hip', 'left_hip', 'left_knee', 'left_ankle', 'right_wrist', 'right_elbow',
        'right_shoulder', 'left_shoulder', 'left_elbow', 'left_wrist', 'head_bottom', 'nose', 'head_top']


def val3_case(n_videos=3, seed=9):
    d = json.load(open(VAL))
    rng = np.random.RandomState(seed)
    by_image = {}
    for a in d['annotations']:
        by_image.setdefault(a['image_id'], []).append(a)
    videos = {}
    for im in d['images']:
        videos.setdefault(os.path.dirname(im['file_name']), []).append(im)
    names = sorted(videos)[:: max(1, len(videos) // n_videos)][:n_videos]
    out = {}
    for vname in names:
        gt, pr = [], []
        frames = [im for im in videos[vname] if im['is_labeled']][:8]
        ids = {}
        for im in frames:
            rects, preds = [], []
            for a in by_image.get(im['id'], []):
                kp = np.asarray(a['keypoints'], np.float64).reshape(17, 3)
                pts = [_pt(j, kp[_VAL_NAMES.index(n), 0], kp[_VAL_NAMES.index(n), 1]) for j, n in enumerate(_DST)
                       if kp[_VAL_NAMES.index(n), 2] > 0]
                hb = a['head_box']
                rects.append({'x1': [hb[0]], 'y1': [hb[1]], 'x2': [hb[2]], 'y2': [hb[3]], 'track_id': [int(a['track_id'])],
                              'annopoints': [{'point': pts}]})
                if rng.rand() < 0.9 and pts:
                    head = np.hypot(hb[2] - hb[0], hb[3] - hb[1])
                    tid = ids.setdefault(int(a['track_id']), int(rng.randint(1000)))
                    if rng.rand() < 0.05:
                        tid = int(rng.randint(1000))             # a swapped id
                    pp = [_pt(p['id'][0], p['x'][0] + rng.normal(0, 0.15 * head), p['y'][0] + rng.normal(0, 0.15 * head),
                              np.round(rng.rand(), 3)) for p in pts if rng.rand() < 0.9]
                    preds.append({'annopoints': [{'point': pp}], 'score': [float(rng.rand())], 'track_id': [tid]})
            for _ in range(rng.randint(0, 3)):                   # false positives
                c = rng.rand(2) * [im['width'], im['height']]
                preds.append({'annopoints': [{'point': [_pt(j, c[0] + rng.normal(0, 20), c[1] + rng.normal(0, 20), np.round(rng.rand(), 3))
                                                        for j in range(J) if rng.rand() < 0.6]}],
                              'score': [float(rng.rand())], 'track_id': [int(rng.randint(1000))]})
            gt.append({'image': [{'name': im['original_file_name']}], 'annorect': rects})
            pr.append({'image': im['original_file_name'], 'annorect': preds})
        out[vname.replace('/', '_') + '.json'] = ({'annolist': gt}, {'annolist': pr})
    return out


sys.path.insert(0, ROOT)
from detectandtrack_b200.datasets import posetrack_synth  # noqa: E402


def cases():
    return {'edge': edge_case(), 'synth': posetrack_synth.make_videos(n_videos=4, frames=16, labelled=10, max_gt=8, max_pr=12, seed=2),
            'val3': val3_case()}


def main():
    arrays = {}
    for case, videos in cases().items():
        files = {'gt': {n: v[0] for n, v in videos.items()}, 'pred': {n: v[1] for n, v in videos.items()}}
        with tempfile.TemporaryDirectory() as tmp:
            res = run_reference(*posetrack_synth.write_dirs(videos, tmp))
        arrays[case + '/files'] = np.array(json.dumps(files))
        for k, v in res.items():
            arrays[case + '/' + k] = v
        print(case, 'mAP %.6f MOTA %.6f' % (res['apAll'][-1, 0], res['metrics'][-4, 0]))
    np.savez_compressed(os.path.join(HERE, 'poseval.npz'), **arrays)


if __name__ == '__main__':
    main()
