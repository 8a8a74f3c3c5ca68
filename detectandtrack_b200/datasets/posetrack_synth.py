"""Seeded synthetic PoseTrack annotation / prediction directories for tests and benchmarks.

    make_videos(n_videos=50, frames=118, labelled=53, max_gt=36, max_pr=60, seed=0) -> {file name: (gt, pred)}
    write_dirs(videos, root) -> (gt_dir, pred_dir)

The default sizes follow PoseTrack v1.0 val (posetrack_val.json: 50 videos, 5906 frames, 2640 labelled, up to 36
people per frame).  Each video has people on random walks with head boxes and 15 joints (some unannotated).  The
predictions are jittered GT with dropped joints, false positives, swapped and re-used track ids, scores on a 1e-3 grid
(ties), a few frames without any prediction rect and a few ignore regions whose corners sit on annotated joints.  The
first labelled frame of every video has GT points and predictions, so each video also evaluates on its own."""
import json
import os
import os.path as osp

import numpy as np

N_JOINTS = 15
# joint offsets from the person's centre, in head sizes (x, y)
_LAYOUT = np.array([[-0.6, 4.0], [-0.6, 2.8], [-0.5, 1.6], [0.5, 1.6], [0.6, 2.8], [0.6, 4.0], [-1.2, 1.4], [-1.0, 0.6],
                    [-0.8, -0.2], [0.8, -0.2], [1.0, 0.6], [1.2, 1.4], [0.0, -0.4], [0.0, -1.0], [0.0, -1.6]])


def _point(j, x, y, score=None):
    p = {'id': [int(j)], 'x': [float(x)], 'y': [float(y)]}
    if score is not None:
        p['score'] = [float(score)]
    return p


def make_video(rng, frames, labelled, max_gt, max_pr, name):
    n_tracks = int(rng.randint(1, max_gt + 1))
    start = rng.rand(n_tracks, 2) * [1200, 600] + [40, 60]
    head = rng.uniform(18, 60, n_tracks)
    step = rng.normal(0, 4, (frames, n_tracks, 2)).cumsum(axis=0)
    tid = rng.choice(1000, n_tracks, replace=False)
    lab = np.sort(rng.choice(frames, min(labelled, frames), replace=False))
    # prediction ids: mostly one per track, some tracks swap ids mid-video, some ids are used twice
    pid = rng.choice(1000, n_tracks, replace=False)
    swap_at = rng.randint(0, frames, n_tracks)
    swap_to = rng.choice(1000, n_tracks)
    gt_list, pr_list = [], []
    for f in range(frames):
        img = 'images/%s/%05d.jpg' % (name, f + 1)
        gt_f = {'image': [{'name': img}], 'imgnum': [f + 1], 'annorect': []}
        pr_f = {'image': img, 'imagenum': [f + 1], 'annorect': []}
        if f in lab:
            visible = rng.rand(n_tracks) < 0.8
            visible[rng.randint(n_tracks)] = True
            for t in np.flatnonzero(visible)[:max_gt]:
                c = start[t] + step[f, t]
                h = head[t]
                hx, hy = c[0] + rng.uniform(-2, 2), c[1] - 1.6 * h
                rect = {'x1': [float(np.round(hx - h / 2, 2))], 'y1': [float(np.round(hy - h / 2, 2))],
                        'x2': [float(np.round(hx + h / 2, 2))], 'y2': [float(np.round(hy + h / 2, 2))],
                        'track_id': [int(tid[t])], 'annopoints': [{'point': []}]}
                xy = np.round(c + _LAYOUT * h * 0.9 + rng.normal(0, 2, (N_JOINTS, 2)), 1)
                has = rng.rand(N_JOINTS) < 0.85
                first = f == lab[0]
                if rng.rand() < 0.03 and not first:
                    has[:] = False                      # a rect whose points list is empty
                for j in np.flatnonzero(has):
                    rect['annopoints'][0]['point'].append(_point(j, xy[j, 0], xy[j, 1]))
                if rng.rand() < 0.02 and not first:
                    del rect['annopoints']              # a rect without points
                gt_f['annorect'].append(rect)
                if (first or rng.rand() < 0.92) and len(pr_f['annorect']) < max_pr:
                    sigma = h * (0.05 if rng.rand() < 0.8 else 0.6)
                    pxy = xy + rng.normal(0, sigma, (N_JOINTS, 2))
                    keep = rng.rand(N_JOINTS) < 0.9
                    ident = int(swap_to[t] if f >= swap_at[t] and rng.rand() < 0.3 else pid[t])
                    points = [_point(j, pxy[j, 0], pxy[j, 1], np.round(rng.rand(), 3)) for j in np.flatnonzero(keep)]
                    pr_f['annorect'].append({'annopoints': [{'point': points}], 'score': [float(rng.rand())],
                                             'track_id': [ident]})
            for _ in range(rng.randint(0, 6)):           # false positives
                if len(pr_f['annorect']) >= max_pr:
                    break
                c = rng.rand(2) * [1280, 720]
                points = [_point(j, c[0] + rng.normal(0, 30), c[1] + rng.normal(0, 30), np.round(rng.rand(), 3))
                          for j in range(N_JOINTS) if rng.rand() < 0.7]
                pr_f['annorect'].append({'annopoints': [{'point': points}], 'score': [float(rng.rand())],
                                         'track_id': [int(rng.choice(1000))]})
            if gt_f['annorect'] and rng.rand() < 0.1 and f != lab[0]:
                # an ignore region: an axis-aligned box with one corner on an annotated joint (on the boundary)
                rect = gt_f['annorect'][0]
                pts = rect.get('annopoints', [{'point': []}])[0]['point']
                if pts:
                    x0, y0 = pts[0]['x'][0], pts[0]['y'][0]
                    w, hh = rng.uniform(10, 80, 2)
                    gt_f['ignore_regions'] = [{'point': [_point(0, x0, y0), _point(1, x0 + w, y0), _point(2, x0 + w, y0 + hh),
                                                         _point(3, x0, y0 + hh)]}]
            if f != lab[0] and rng.rand() < 0.04:
                pr_f['annorect'] = []                   # no prediction at all: MOT inputs of the previous frame
        gt_list.append(gt_f)
        pr_list.append(pr_f)
    return {'annolist': gt_list}, {'annolist': pr_list}


def make_videos(n_videos=50, frames=118, labelled=53, max_gt=36, max_pr=60, seed=0):
    rng = np.random.RandomState(seed)
    return {'%06d_mpii_test.json' % (10000 + v): make_video(rng, frames, labelled, max_gt, max_pr, '%06d_mpii_test' % (10000 + v))
            for v in range(n_videos)}


def write_dirs(videos, root):
    gt_dir, pred_dir = osp.join(root, 'gt') + os.sep, osp.join(root, 'pred') + os.sep
    os.makedirs(gt_dir, exist_ok=True)
    os.makedirs(pred_dir, exist_ok=True)
    for name, (gt, pr) in videos.items():
        with open(osp.join(gt_dir, name), 'w') as f:
            json.dump(gt, f)
        with open(osp.join(pred_dir, name), 'w') as f:
            json.dump(pr, f)
    return gt_dir, pred_dir
