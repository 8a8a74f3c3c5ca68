"""GPU: the device PoseTrack evaluation (csrc/poseval.cu behind datasets/posetrack_eval.py) against the oracle
(oracle/poseval.py): per-(prediction, joint) labels, per-(frame, joint) GT counts and per-(sequence, joint) CLEAR-MOT
event counts exactly; sumD, AP, precision, recall and the final tables within 1e-12 relative; the per-video scores;
the golden cases of tests/golden/poseval.npz; and tools/test_net.py -> tools/compute_tracks.py with an annotation
directory end to end."""
import copy
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from detectandtrack_b200.datasets import posetrack_eval as E
from detectandtrack_b200.datasets import posetrack_synth as S
from oracle import poseval as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
J = 15


def _close(a, b, rel=1e-12):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    same_nan = np.isnan(a) == np.isnan(b)
    assert same_nan.all(), (a, b)
    m = ~np.isnan(a)
    assert np.array_equal(np.isinf(a[m]), np.isinf(b[m])), (a, b)
    f = m & ~np.isinf(a)
    assert np.all(np.abs(a[f] - b[f]) <= rel * np.maximum(np.abs(b[f]), 1e-300) + 1e-300), (a[f] - b[f], b[f])


def check_dirs(gt_dir, pred_dir, per_video=True):
    """Device vs oracle on one directory pair; returns the device result."""
    gt, pr, names = E.load_data_dir(gt_dir, pred_dir)
    ogt, opr, _ = O.load_data_dir(gt_dir, pred_dir)
    assert gt == ogt and pr == opr
    pack = E.PoseTrackPack(gt, pr, names)
    res = E.evaluate_pack(pack, True, True, per_video)
    raw = res['raw']
    scoresAll, labelsAll, nGTall, motAll = O.assign_gt_multi(copy.deepcopy(ogt), copy.deepcopy(opr))
    # labels of every predicted joint, in the reference's concatenation order
    present = pack.pr_kp[:, :, 3] != 0
    for j in range(J):
        dev = raw['labels'][present[:, j], j]
        ref = np.array([l for f in range(pack.nframes) for l in labelsAll[j][f]], np.int64)
        assert np.array_equal(dev.astype(np.int64), ref), j
        assert np.array_equal(raw['ngt'][j, :pack.nframes], nGTall[j].astype(np.int64)), j
    # per-joint AP / precision / recall of all frames
    apAll, preAll, recAll = O.ap_metrics(scoresAll, labelsAll, nGTall)
    _close(raw['ap'][:J, 0], apAll[:J, 0])
    _close(raw['ap'][:J, 1], preAll[:J, 0])
    _close(raw['ap'][:J, 2], recAll[:J, 0])
    for mine, ref in zip(res['ap'], (apAll, preAll, recAll)):
        _close(mine, ref)
    # per-(sequence, joint) events
    seqs = O.sequences(ogt)
    per_seq = [O.mot_sequence_counts(frames, motAll) for _, frames in seqs]
    n_all = len(seqs)
    assert [k for k in raw['lists'] if k[0] == 'all'] == [('all', s) for s, _ in seqs]
    assert np.array_equal(raw['counts'][:n_all], np.stack([c for c, _ in per_seq]))
    _close(raw['sumd'][:n_all], np.stack([d for _, d in per_seq]))
    _close(res['metrics'], O.mot_metrics([c for c, _ in per_seq], [d for _, d in per_seq]))
    if per_video:
        ref = O.evaluate_per_video(gt_dir, pred_dir)
        got = {os.path.basename(names[s]): v for s, v in res['videos'].items()}
        assert set(got) <= set(ref)
        for k in ref:
            _close(got.get(k, (0.0, np.nan)), ref[k])
    return res


def test_val_scale_synthetic(tmp_path):
    """50 videos x 118 frames (53 labelled), up to 36 GT and 60 predictions per frame."""
    gt_dir, pred_dir = S.write_dirs(S.make_videos(seed=0), str(tmp_path))
    res = check_dirs(gt_dir, pred_dir)
    assert np.isfinite(res['ap'][0][-1, 0]) and np.isfinite(res['metrics'][-4, 0])


@pytest.mark.parametrize('seed', [1, 2, 3])
def test_small_synthetic(tmp_path, seed):
    gt_dir, pred_dir = S.write_dirs(S.make_videos(n_videos=4, frames=20, labelled=12, seed=seed), str(tmp_path))
    check_dirs(gt_dir, pred_dir)


def test_full_frames_at_the_limits(tmp_path):
    """64 GT and 224 predictions in a frame: the largest assignment and MOT tiles."""
    videos = S.make_videos(n_videos=2, frames=4, labelled=4, max_gt=64, max_pr=224, seed=7)
    for name, (gt, pr) in videos.items():                 # pad every labelled frame to 224 predictions
        for f in pr['annolist']:
            while f['annorect'] and len(f['annorect']) < 224:
                r = copy.deepcopy(f['annorect'][len(f['annorect']) % 5])
                r['track_id'] = [len(f['annorect']) % 1000]
                f['annorect'].append(r)
    gt_dir, pred_dir = S.write_dirs(videos, str(tmp_path))
    check_dirs(gt_dir, pred_dir)
    pack = E.PoseTrackPack(*E.load_data_dir(gt_dir, pred_dir))
    assert pack.max_pr == 224


def _stale_dirs(root, first_has_predictions=True):
    videos = S.make_videos(n_videos=3, frames=10, labelled=8, seed=11)
    names = sorted(videos)
    # the second video's first labelled frame has no prediction: in the full evaluation it reuses the last MOT inputs
    # of the first video; alone, the video cannot be scored
    gt, pr = videos[names[1]]
    first = [i for i, f in enumerate(gt['annolist']) if f['annorect']][0]
    pr['annolist'][first]['annorect'] = []
    if not first_has_predictions:
        gt, pr = videos[names[0]]
        first = [i for i, f in enumerate(gt['annolist']) if f['annorect']][0]
        pr['annolist'][first]['annorect'] = []
    return S.write_dirs(videos, root)


def test_stale_mot_inputs_cross_sequences(tmp_path):
    gt_dir, pred_dir = _stale_dirs(str(tmp_path))
    res = check_dirs(gt_dir, pred_dir)
    vids = sorted(res['videos'].items())
    assert np.isnan(vids[1][1][0]) and np.isnan(vids[1][1][1])
    assert all(np.isfinite(v[1][0]) for k, v in enumerate(vids) if k != 1)


def test_no_earlier_mot_inputs_is_an_error(tmp_path):
    gt_dir, pred_dir = _stale_dirs(str(tmp_path), first_has_predictions=False)
    with pytest.raises(ValueError, match='has no MOT inputs'):
        E.evaluate(gt_dir, pred_dir, verbose=False)
    (ap, _, _), metrics = E.evaluate(gt_dir, pred_dir, eval_track=False, verbose=False)   # the AP alone is fine
    assert np.isfinite(ap[-1, 0]) and np.isnan(metrics).all()


Z = np.load(os.path.join(GOLDEN, 'poseval.npz'))


@pytest.mark.parametrize('case', sorted({k.split('/')[0] for k in Z.files}))
def test_golden_case(case, tmp_path):
    files = json.loads(str(Z[case + '/files']))
    gt_dir, pred_dir = S.write_dirs({n: (files['gt'][n], files['pred'][n]) for n in files['gt']}, str(tmp_path))
    res = check_dirs(gt_dir, pred_dir, per_video=False)
    _close(res['ap'][0], Z[case + '/apAll'])
    _close(res['ap'][1], Z[case + '/preAll'])
    _close(res['ap'][2], Z[case + '/recAll'])
    _close(res['metrics'], Z[case + '/metrics'])
    n = len(Z[case + '/seq_counts'])
    assert np.array_equal(res['raw']['counts'][:n], Z[case + '/seq_counts'])
    _close(res['raw']['sumd'][:n], Z[case + '/seq_sumd'])


def test_eval_posetrack_cli_prints_the_tables(tmp_path):
    gt_dir, pred_dir = S.write_dirs(S.make_videos(n_videos=2, frames=8, labelled=6, seed=5), str(tmp_path))
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'eval_posetrack.py'), '-g', gt_dir, '-p', pred_dir, '-e', '-t'],
                       env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    (ap, _, _), metrics = O.evaluate(gt_dir, pred_dir)
    assert E.get_format_row(E.get_cum(ap)) in r.stdout
    assert E.get_format_row(E.get_cum(metrics)) in r.stdout
    assert E.get_mot_header() in r.stdout and E.get_header() in r.stdout


def _e2e_yaml():
    """The synthetic keypoint R-CNN config of tests/test_gpu_tools.py."""
    import importlib.util
    spec = importlib.util.spec_from_file_location('_gpu_tools_cfg', os.path.join(ROOT, 'tests', 'test_gpu_tools.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.YAML


def _annotations(root, videos=2, frames=3, h=96, w=128, seed=3):
    """GT JSON named like the writer's files for synthetic_<videos>x<frames>_<h>x<w>: a few people per frame."""
    rng = np.random.RandomState(seed)
    os.makedirs(root, exist_ok=True)
    for v in range(videos):
        annolist = []
        tracks = rng.rand(4, 2) * [w - 30, h - 40] + [15, 20]
        for f in range(frames):
            rects = []
            for t in range(4):
                c = tracks[t] + rng.normal(0, 2, 2)
                hs = 10.0
                pts = [{'id': [j], 'x': [float(c[0] + rng.normal(0, 8))], 'y': [float(c[1] + rng.normal(0, 12))]}
                       for j in range(J) if rng.rand() < 0.9]
                rects.append({'x1': [float(c[0] - hs / 2)], 'y1': [float(c[1] - 20 - hs / 2)], 'x2': [float(c[0] + hs / 2)],
                              'y2': [float(c[1] - 20 + hs / 2)], 'track_id': [t], 'annopoints': [{'point': pts}]})
            annolist.append({'image': [{'name': 'synthetic/vid%03d/%06d.jpg' % (v, f)}], 'annorect': rects})
        with open(os.path.join(root, 'synthetic_vid%03d.json' % v), 'w') as fo:
            json.dump({'annolist': annolist}, fo)
    return root + os.sep


def test_test_net_then_compute_tracks_scores_the_videos(tmp_path):
    cfg = tmp_path / 'cfg.yaml'
    cfg.write_text(_e2e_yaml())
    out = str(tmp_path / 'out')
    annot = _annotations(str(tmp_path / 'annot'))
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'test_net.py'), '--cfg', str(cfg), 'OUTPUT_DIR', out],
                       env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'compute_tracks.py'), '--cfg', str(cfg), 'OUTPUT_DIR', out,
                        'EVAL.POSETRACK_ANNOTATION_DIR', annot, 'EVAL.EVAL_MPII_PER_VIDEO', 'True',
                        'EVAL.EVAL_MPII_DROP_DETECTION_THRESHOLD', '0.0'],
                       env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    m = re.search(r'\(total mAP, total MOTA\) = \(([^,]+), ([^)]+)\)', r.stdout + r.stderr)
    assert m, r.stdout[-3000:] + r.stderr[-3000:]
    ddir = os.path.join(out, 'test', 'synthetic_2x3_96x128', 'keypoint_rcnn')
    json_dir = os.path.join(ddir, 'detections_withTracks.pkl_json') + os.sep
    (ap, _, _), metrics = O.evaluate(annot, json_dir)
    _close([float(m.group(1)), float(m.group(2))], [ap[-1, 0], metrics[-4, 0]])
    per = O.evaluate_per_video(annot, json_dir)
    want = sorted([('synthetic/vid%03d' % v,) + per['synthetic_vid%03d.json' % v] for v in range(2)], key=lambda x: x[1])
    got = [l.split(' ') for l in open(os.path.join(ddir, 'detections_withTracks.pkl_per_video_scores.txt')).read().splitlines()]
    assert [g[0] for g in got] == [w[0] for w in want]
    _close([[float(g[1]), float(g[2])] for g in got], [[w[1], w[2]] for w in want])
