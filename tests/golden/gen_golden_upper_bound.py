"""Golden vectors for the upper-bound experiments (TRACKING.DEBUG.UPPER_BOUND*, poseval's computeUpperBound), from the
REFERENCE's own source.

    python tests/golden/gen_golden_upper_bound.py      -> tests/golden/upper_bound.npz

Tracking, from lib/core/tracking_engine.py's source text (the module imports Caffe2-era code): _get_boxes ... _set_boxes
(:70-84), _compute_pairwise_iou / _compute_pairwise_kpt_distance (:106-129), _compute_distance_matrix ...
_compute_tracks_video (:158-350), with lib/utils/keypoints.py:266-291 for the pose-pck cost and lib/utils/boxes.py's
bbox_overlaps over the reference's own cython_bbox (oracle/build_ref.py).  Shims: cfg is a namespace with the keys the
code reads; img_utils.get_image_path returns entry['image']; the logger is silent.

Tracking cases: four seeded synthetic videos (ties, empty-GT frames, frames without detections, G > |D| and G < |D|),
then three videos of real GT from PoseTrack v1.0 val with jittered, dropped, false-positive and duplicated detections.
Tracking case t<k> (one video, every mode of MODES with pose-pck weight 0 and 1, hungarian and greedy): inputs boxes
[F, Dmax, 5], poses [F, Dmax, 4, 17], counts [F], gt_boxes [F, Gmax, 4], gt_kps [F, Gmax, 3, 17] int32, gt_tracks
[F, Gmax], gt_counts [F]; per mode m<j>: out_boxes, out_poses, out_counts, out_tracks (as the inputs, -1 padded).

Evaluation: the poseval cases of gen_golden_poseval.py (edge, synth, val3) through evaluateTracking(..., True): metrics
[19, 1], seq_counts [S, 15, 4] and seq_sumd [S, 15] per case under 'u_<case>/'.
"""
import copy
import json
import os
import sys
import tempfile
import types

import numpy as np
import scipy.optimize

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = '/root/reference/lib/'
VAL = '/root/reference/lib/datasets/lists/PoseTrack/v1.0/posetrack_val.json'
K = 17
NAMES = ['nose', 'head_bottom', 'head_top', 'left_ear', 'right_ear', 'left_shoulder', 'right_shoulder', 'left_elbow',
         'right_elbow', 'left_wrist', 'right_wrist', 'left_hip', 'right_hip', 'left_knee', 'right_knee', 'left_ankle',
         'right_ankle']
# (UPPER_BOUND, _2_GT_KPS, _2_GT_KPS_ONLY_CONF, _5_GT_KPS_ONLY)
MODES = [(1, 0, 0, 0), (1, 1, 0, 0), (1, 1, 1, 0), (0, 0, 0, 1), (1, 0, 0, 1), (1, 1, 0, 1)]
SETTINGS = [(w, algo) for w in (0.0, 1.0) for algo in ('hungarian', 'greedy')]


def _lines(path, a, b):
    return '\n'.join(open(path).read().split('\n')[a - 1:b])


def tracking_reference(mode, w_pck, algo):
    sys.path.insert(0, ROOT)
    from oracle import build_ref
    assert build_ref.build(), 'reference not present'
    from oracle._ref import cython_bbox
    ub, ub2, conf, ub5 = (bool(x) for x in mode)
    cfg = types.SimpleNamespace(
        TRACKING=types.SimpleNamespace(
            DEBUG=types.SimpleNamespace(UPPER_BOUND=ub, UPPER_BOUND_2_GT_KPS=ub2, UPPER_BOUND_2_GT_KPS_ONLY_CONF=conf,
                                        UPPER_BOUND_3_SHOTS=False, UPPER_BOUND_5_GT_KPS_ONLY=ub5),
            DISTANCE_METRICS=('bbox-overlap', 'cnn-cosdist', 'pose-pck'), DISTANCE_METRIC_WTS=(1.0, 0.0, w_pck),
            BIPARTITE_MATCHING_ALGO=algo))
    bns = {'np': np, 'cfg': cfg, 'cython_bbox_overlaps': cython_bbox.bbox_overlaps}
    exec(_lines(REF + 'utils/boxes.py', 26, 71), bns)
    kps_utils = types.ModuleType('kps_utils')
    kps_utils.np = np
    exec(_lines(REF + 'utils/keypoints.py', 266, 291), kps_utils.__dict__)
    ns = {'np': np, 'scipy': scipy, 'cfg': cfg, 'box_utils': types.SimpleNamespace(bbox_overlaps=bns['bbox_overlaps']),
          'kps_utils': kps_utils, 'img_utils': types.SimpleNamespace(get_image_path=lambda e: e['image']),
          'logger': types.SimpleNamespace(warning=lambda *a: None), 'MAX_TRACK_IDS': 999, 'FIRST_TRACK_ID': 0}
    src = REF + 'core/tracking_engine.py'
    for a, b in ((70, 84), (106, 129), (158, 350)):
        exec(_lines(src, a, b), ns)
    return ns['_compute_tracks_video']


def _video(rng, F, n_people=6, empty_gt=(), no_dets=(), ties=(), fp=2):
    """GT people moving across frames; detections are jittered GT with drops, false positives and exact duplicates."""
    W, H = 640.0, 480.0
    c0 = rng.uniform([60, 60], [W - 60, H - 60], (n_people, 2))
    size = rng.uniform([30, 60], [80, 160], (n_people, 2))
    frames = []
    for f in range(F):
        c = c0 + f * rng.normal(0, 6, (n_people, 2))
        present = rng.rand(n_people) < 0.85
        if f in empty_gt:
            present[:] = False
        ids = np.flatnonzero(present)
        gb = np.stack([c[ids, 0] - size[ids, 0] / 2, c[ids, 1] - size[ids, 1] / 2,
                       c[ids, 0] + size[ids, 0] / 2, c[ids, 1] + size[ids, 1] / 2], 1).astype(np.float32).reshape(-1, 4)
        gk = np.zeros((len(ids), 3, K), np.int32)
        for i, p in enumerate(ids):
            gk[i, 0] = np.round(c[p, 0] + rng.uniform(-size[p, 0] / 2, size[p, 0] / 2, K))
            gk[i, 1] = np.round(c[p, 1] + rng.uniform(-size[p, 1] / 2, size[p, 1] / 2, K))
            gk[i, 2] = rng.randint(0, 3, K)
        gt = (ids * 7 + 3).astype(np.int64)
        db, dp = [], []
        if f not in no_dets:
            for i in range(len(ids)):
                if rng.rand() < 0.15:
                    continue
                db.append(np.r_[gb[i] + rng.normal(0, 4, 4), rng.uniform(0.5, 1)])
                p = np.zeros((4, K))
                p[:2] = gk[i, :2] + rng.normal(0, 4, (2, K))
                p[2] = rng.normal(1, 2, K)
                p[3] = rng.uniform(0, 1, K)
                dp.append(p)
            for _ in range(rng.randint(0, fp + 1)):
                xy = rng.uniform([0, 0], [W - 80, H - 120])
                db.append(np.r_[xy, xy + rng.uniform(30, 100, 2), rng.uniform(0.5, 1)])
                p = np.zeros((4, K))
                p[0] = xy[0] + rng.uniform(0, 60, K)
                p[1] = xy[1] + rng.uniform(0, 90, K)
                p[2:] = rng.uniform(0, 1, (2, K))
                dp.append(p)
            if f in ties and db:
                db.append(db[0].copy())
                dp.append(dp[0].copy())
            order = rng.permutation(len(db))
            db = [db[i] for i in order]
            dp = [dp[i] for i in order]
        frames.append((np.array(db, np.float32).reshape(-1, 5), [p.astype(np.float32) for p in dp], gb, gk, gt))
    return frames


def _val_videos(rng, n_videos=3, n_frames=6):
    """Real GT from PoseTrack v1.0 val (the file gen_golden_poseval.py reads): labelled frames of a few videos, boxes
    xywh -> xyxy (x2 = x + w - 1, as json_dataset), keypoints truncated to int32 (json_dataset's array), track ids; the
    detections are jittered GT with drops, false positives and a duplicate."""
    d = json.load(open(VAL))
    by_image = {}
    for a in d['annotations']:
        by_image.setdefault(a['image_id'], []).append(a)
    videos = {}
    for im in d['images']:
        videos.setdefault(os.path.dirname(im['file_name']), []).append(im)
    names = sorted(videos)[1::max(1, len(videos) // n_videos)][:n_videos]
    out = []
    for vname in names:
        frames = []
        for f, im in enumerate([im for im in videos[vname] if im['is_labeled']][:n_frames]):
            anns = [a for a in by_image.get(im['id'], []) if a.get('bbox') and len(a['bbox']) == 4]
            gb = np.array([[a['bbox'][0], a['bbox'][1], a['bbox'][0] + a['bbox'][2] - 1, a['bbox'][1] + a['bbox'][3] - 1]
                           for a in anns], np.float32).reshape(-1, 4)
            kp = np.zeros((len(anns), 3, K), np.int32)
            for i, a in enumerate(anns):
                kp[i] = np.asarray(a['keypoints'], np.float64).reshape(K, 3).T
            gt = np.array([a['track_id'] for a in anns], np.int64)
            frames.append((gb, kp, gt) + _dets_from_gt(rng, gb, kp, im['width'], im['height'], ties=(f == 1), fp=3))
        out.append([(db, dp, gb, gk, gt) for gb, gk, gt, db, dp in frames])
    return out


def _dets_from_gt(rng, gb, gk, W, H, ties=False, fp=2):
    db, dp = [], []
    scale = np.maximum(gb[:, 2:] - gb[:, :2], 8) if len(gb) else np.zeros((0, 2))
    for i in range(len(gb)):
        if rng.rand() < 0.15:
            continue
        db.append(np.r_[gb[i] + rng.normal(0, 0.05, 4) * np.r_[scale[i], scale[i]], rng.uniform(0.5, 1)])
        p = np.zeros((4, K))
        p[:2] = gk[i, :2] + rng.normal(0, 0.04 * scale[i].mean(), (2, K))
        p[2] = rng.normal(1, 2, K)
        p[3] = rng.uniform(0, 1, K)
        dp.append(p)
    for _ in range(rng.randint(0, fp + 1)):
        xy = rng.uniform([0, 0], [W - 100, H - 150])
        db.append(np.r_[xy, xy + rng.uniform(40, 100, 2), rng.uniform(0.5, 1)])
        p = np.zeros((4, K))
        p[0] = xy[0] + rng.uniform(0, 60, K)
        p[1] = xy[1] + rng.uniform(0, 90, K)
        p[2:] = rng.uniform(0, 1, (2, K))
        dp.append(p)
    if ties and db:
        db.append(db[0].copy())
        dp.append(dp[0].copy())
    order = rng.permutation(len(db))
    return np.array([db[i] for i in order], np.float32).reshape(-1, 5), [dp[i].astype(np.float32) for i in order]


def tracking_cases():
    rng = np.random.RandomState(20261017)
    return [_video(rng, 8, empty_gt=(3,), ties=(1, 5)),                    # G > |D| in frames with drops
            _video(rng, 6, n_people=3, fp=4, no_dets=(2,), ties=(0,)),      # G < |D|: false positives
            _video(rng, 5, n_people=9, empty_gt=(0, 4)),
            _video(rng, 1, n_people=4, ties=(0,))] + _val_videos(np.random.RandomState(7))


def _pad(arrs, shape, dtype, fill=0):
    n = max([len(a) for a in arrs] + [1])
    out = np.full((len(arrs), n) + shape, fill, dtype)
    for f, a in enumerate(arrs):
        if len(a):
            out[f, :len(a)] = np.asarray(a).reshape((len(a),) + shape)
    return out


def run_tracking(frames, mode, w_pck, algo):
    fn = tracking_reference(mode, w_pck, algo)
    dets = {'all_boxes': [[], [fr[0].copy() for fr in frames]], 'all_keyps': [[], [[p.copy() for p in fr[1]] for fr in frames]]}
    ds = types.SimpleNamespace(person_cat_info={'keypoints': NAMES})
    video = [({'image': 'vid/%05d.jpg' % f, 'boxes': fr[2].copy(), 'gt_keypoints': fr[3].copy(), 'tracks': fr[4].copy(),
               'dataset': ds}, f) for f, fr in enumerate(frames)]
    tracks = fn(video, dets)
    return dets['all_boxes'][1], dets['all_keyps'][1], tracks


def tracking_arrays():
    out = {}
    for k, frames in enumerate(tracking_cases()):
        t = 't%d_' % k
        out[t + 'boxes'] = _pad([fr[0] for fr in frames], (5,), np.float32)
        out[t + 'poses'] = _pad([fr[1] for fr in frames], (4, K), np.float32)
        out[t + 'counts'] = np.array([len(fr[0]) for fr in frames], np.int32)
        out[t + 'gt_boxes'] = _pad([fr[2] for fr in frames], (4,), np.float32)
        out[t + 'gt_kps'] = _pad([fr[3] for fr in frames], (3, K), np.int32)
        out[t + 'gt_tracks'] = _pad([fr[4] for fr in frames], (), np.int64, -1)
        out[t + 'gt_counts'] = np.array([len(fr[2]) for fr in frames], np.int32)
        j = 0
        for mode in MODES:
            for w, algo in SETTINGS:
                b, p, tr = run_tracking(frames, mode, w, algo)
                m = t + 'm%d_' % j
                out[m + 'params'] = np.array(list(mode) + [w, algo == 'greedy'], np.float64)
                assert all(x.dtype == np.float32 for x in b) and all(x.dtype == np.float32 for ps in p for x in ps)
                out[m + 'out_boxes'] = _pad(b, (5,), np.float32)
                out[m + 'out_poses'] = _pad(p, (4, K), np.float32)
                out[m + 'out_counts'] = np.array([len(x) for x in b], np.int32)
                out[m + 'out_tracks'] = _pad(tr, (), np.int64, -1)
                assert [len(x) for x in tr] == [len(x) for x in b]
                j += 1
    return out


def eval_arrays():
    sys.path.insert(0, HERE)
    import gen_golden_poseval as G
    from detectandtrack_b200.datasets import posetrack_synth
    out = {}
    J = G.J
    for case, videos in G.cases().items():
        eh, ap_ns, tr_ns = G.reference()
        with tempfile.TemporaryDirectory() as tmp:
            gt_dir, pr_dir = posetrack_synth.write_dirs(videos, tmp)
            gtFramesAll, prFramesAll = eh.load_data_dir(['', gt_dir, pr_dir])
        metricsAll = tr_ns['evaluateTracking'](copy.deepcopy(gtFramesAll), copy.deepcopy(prFramesAll), True)
        metrics = np.full((J + 4, 1), np.nan)
        for i in range(J + 1):
            metrics[i, 0] = metricsAll['mota'][0, i]
        metrics[J + 1, 0], metrics[J + 2, 0], metrics[J + 3, 0] = (metricsAll[k][0, J] for k in ('motp', 'pre', 'rec'))
        _, _, _, motAll = eh.assignGTmulti(copy.deepcopy(gtFramesAll), copy.deepcopy(prFramesAll), 0.5, True)
        seqidxs = np.array([f['seq_id'] for f in gtFramesAll])
        uniq = np.unique(seqidxs)
        names = ['num_misses', 'num_switches', 'num_false_positives', 'num_objects', 'num_detections']
        counts, sumd = np.zeros((len(uniq), J, 4), np.int64), np.zeros((len(uniq), J))
        for si in range(len(uniq)):
            _, accs = tr_ns['process_frame'](si, J, seqidxs, uniq, motAll, names)
            for i in range(J):
                df = accs[i].events.frame()
                counts[si, i] = [(df.Type == t).sum() for t in ('MATCH', 'SWITCH', 'FP', 'MISS')]
                sumd[si, i] = accs[i].events['D'].sum()
        out['u_%s/metrics' % case], out['u_%s/seq_counts' % case], out['u_%s/seq_sumd' % case] = metrics, counts, sumd
        print(case, '-u MOTA %.6f' % metrics[-4, 0])
    return out


def main():
    out = tracking_arrays()
    out.update(eval_arrays())
    path = os.path.join(HERE, 'upper_bound.npz')
    np.savez_compressed(path, **out)
    print('wrote upper_bound.npz: %d arrays, %d bytes' % (len(out), os.path.getsize(path)))


if __name__ == '__main__':
    main()
