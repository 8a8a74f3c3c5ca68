"""CPU: the PoseTrack evaluation's host side and oracle.
  - oracle/poseval.py equals the reference's own poseval (tests/golden/poseval.npz, gen_golden_poseval.py) on every golden
    case: labels, GT counts and per-(sequence, joint) events exactly; AP, MOTA, MOTP and sumD to 1e-12 relative;
  - the host loader (datasets/posetrack_eval.load_data_dir) equals the reference's load_data_dir result;
  - the exact ignore-region test, the size limits and the errors, and the C ABI's argument checks, without a GPU."""
import atexit
import ctypes as C
import json
import os
import shutil
import tempfile

import numpy as np
import pytest

from detectandtrack_b200 import _lib as L
from detectandtrack_b200.datasets import posetrack_eval as E
from detectandtrack_b200.datasets import posetrack_synth as S
from oracle import poseval as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
Z = np.load(os.path.join(GOLDEN, 'poseval.npz'))
CASES = sorted({k.split('/')[0] for k in Z.files})
J = 15


def _dirs(case, _made={}):
    """The golden case's GT and prediction directories, written once from poseval.npz."""
    if case not in _made:
        files = json.loads(str(Z[case + '/files']))
        root = tempfile.mkdtemp(prefix='poseval_%s_' % case)
        atexit.register(shutil.rmtree, root, True)
        _made[case] = S.write_dirs({n: (files['gt'][n], files['pred'][n]) for n in files['gt']}, root)
    return _made[case]


def _close(a, b, rel=1e-12):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape
    assert np.array_equal(np.isnan(a), np.isnan(b)), (a, b)
    m = ~np.isnan(a)
    assert np.array_equal(a[m & np.isinf(a)], b[m & np.isinf(a)]), (a, b)
    f = m & ~np.isinf(a)
    assert np.all(np.abs(a[f] - b[f]) <= rel * np.abs(b[f])), (a[f], b[f])


def test_golden_cases_present():
    assert CASES == ['edge', 'synth', 'val3']


@pytest.mark.parametrize('case', CASES)
def test_oracle_equals_reference(case):
    gt, pr, _ = O.load_data_dir(*_dirs(case))
    ap, metrics, per_seq = O.evaluate_frames(gt, pr)
    for k, v in zip(('apAll', 'preAll', 'recAll'), ap):
        _close(v, Z[case + '/' + k])
    _close(metrics, Z[case + '/metrics'])
    assert np.array_equal(np.stack([c for c, _ in per_seq]), Z[case + '/seq_counts'])
    _close(np.stack([d for _, d in per_seq]), Z[case + '/seq_sumd'])
    _, labelsAll, nGTall, _ = O.assign_gt_multi(*O.load_data_dir(*_dirs(case))[:2])
    off = Z[case + '/labels_off']
    for j in range(J):
        got = np.array([l for f in range(nGTall.shape[1]) for l in labelsAll[j][f]], np.int64)
        assert np.array_equal(got, Z[case + '/labels'][off[j]:off[j + 1]]), j
    assert np.array_equal(nGTall.astype(np.int64), Z[case + '/ngt'])


def test_golden_edge_case_covers_the_corners():
    """The hand-made case holds what it claims: a joint with no GT (0/0), stale frames, ignore regions, switches."""
    gt, pr, _ = O.load_data_dir(*_dirs('edge'))
    assert np.isnan(Z['edge/apAll'][7, 0]) and Z['edge/ngt'][7].sum() == 0
    assert Z['edge/seq_counts'][:, :, 1].sum() > 0                         # switches
    assert any(len(p['annorect']) == 0 and len(g['annorect']) > 0 for g, p in zip(gt, pr))       # stale MOT inputs
    assert any(len(g['annorect']) == 0 for g in gt)                        # a GT frame left without people
    assert any('ignore_regions' in g for g in gt)


@pytest.mark.parametrize('case', CASES)
def test_loader_equals_reference_load_data_dir(case):
    gt, pr, names = E.load_data_dir(*_dirs(case))
    want = json.loads(str(Z[case + '/loaded']))
    assert json.loads(json.dumps([gt, pr])) == want
    assert [os.path.basename(n) for n in names] == sorted(os.listdir(_dirs(case)[0]))


def test_pack_layout():
    gt, pr, names = E.load_data_dir(*_dirs('val3'))
    pack = E.PoseTrackPack(gt, pr, names)
    assert pack.nframes == len(gt) and pack.gt_off[-1] == sum(len(f['annorect']) for f in gt)
    assert pack.gt_kp.shape == (pack.gt_off[-1], J, 3) and pack.pr_kp.shape == (pack.pr_off[-1], J, 4)
    assert pack.gt_rect.dtype == np.float64 and pack.pr_kp.dtype == np.float64
    r = gt[0]['annorect'][0]
    assert tuple(pack.gt_rect[0]) == (r['x1'][0], r['y1'][0], r['x2'][0], r['y2'][0])
    assert pack.gt_tid[0] == r['track_id'][0]
    for p in r['annopoints'][0]['point']:
        assert tuple(pack.gt_kp[0, p['id'][0]]) == (p['x'][0], p['y'][0], 1.0)
    assert np.array_equal(pack.pair_off[1:] - pack.pair_off[:-1], pack.n_gt * pack.n_pr)
    assert [s for s, _, _ in pack.seq_ranges()] == sorted(set(pack.seq_id.tolist()))


def test_mot_sources_keep_the_stale_inputs():
    gt, pr, names = E.load_data_dir(*_dirs('edge'))
    pack = E.PoseTrackPack(gt, pr, names)
    src = E.mot_sources(pack)
    stale = np.flatnonzero(~pack.has_mot)
    assert len(stale) and np.all(src[stale] < stale) and np.all(src[pack.has_mot] == np.flatnonzero(pack.has_mot))
    # the first frame of the third sequence takes the second sequence's inputs; alone, it has none
    s, a, b = pack.seq_ranges()[2]
    assert not pack.has_mot[a] and src[a] < a and E.mot_sources(pack, a, b)[0] == -1


def test_polygon_contains_is_exact():
    rng = np.random.RandomState(0)
    for _ in range(30):
        poly = rng.randint(0, 20, (int(rng.randint(3, 8)), 2)).astype(np.float64)
        pts = np.concatenate([np.round(rng.rand(40, 2) * 20, 1), poly,                      # vertices
                              (poly + np.roll(poly, -1, 0)) / 2,                             # edge midpoints (exact)
                              poly + 1e-13, np.round(rng.rand(20, 2) * 20, 1) + 0.1])
        got = E.polygon_contains(poly, pts)
        want = [O.polygon_contains(poly.tolist(), x, y) for x, y in pts]
        assert got.tolist() == want
        assert not got[40:40 + 2 * len(poly)].any()                 # the boundary is outside
    assert not E.polygon_contains([[0, 0], [3, 0], [0, 3]], [[1, 0]])[0]
    assert E.polygon_contains([[0, 0], [3, 0], [0, 3]], [[1, 1]])[0]
    with pytest.raises(ValueError, match='at least 3'):
        E.polygon_contains([[0, 0], [1, 1]], [[0.5, 0.5]])


def _write(tmp_path, videos):
    return S.write_dirs(videos, str(tmp_path))


def test_loader_errors(tmp_path):
    videos = S.make_videos(n_videos=2, frames=4, labelled=3, max_gt=3, max_pr=4, seed=1)
    gt_dir, pred_dir = _write(tmp_path / 'ok', videos)
    os.remove(os.path.join(pred_dir, sorted(videos)[1]))
    with pytest.raises(IOError, match='does not exist'):
        E.load_data_dir(gt_dir, pred_dir)
    bad = json.loads(json.dumps(videos))
    name = sorted(bad)[0]
    bad[name][1]['annolist'].pop()
    gt_dir, pred_dir = _write(tmp_path / 'frames', bad)
    with pytest.raises(ValueError, match=r'# prediction frames 3 <> # GT frames 4 for'):
        E.load_data_dir(gt_dir, pred_dir)
    bad = json.loads(json.dumps(videos))
    rect = [f for f in bad[name][0]['annolist'] if f['annorect']][0]['annorect'][0]
    rect['track_id'] = [1000]
    gt_dir, pred_dir = _write(tmp_path / 'ids', bad)
    with pytest.raises(ValueError, match='track id 1000'):
        E.load_data_dir(gt_dir, pred_dir)
    bad = json.loads(json.dumps(videos))
    frame = [f for f in bad[name][0]['annolist'] if f['annorect']][0]
    frame['ignore_regions'] = [{'point': [{'id': [0], 'x': [0.0], 'y': [0.0]}, {'id': [1], 'x': [1.0], 'y': [1.0]}]}]
    gt_dir, pred_dir = _write(tmp_path / 'poly', bad)
    with pytest.raises(ValueError, match='at least 3'):
        E.load_data_dir(gt_dir, pred_dir)
    with pytest.raises(NotImplementedError):
        E.evaluate(*_dirs('synth'), eval_upper_bound=True)


def test_limits_are_checked_before_any_device_call(tmp_path):
    videos = S.make_videos(n_videos=1, frames=2, labelled=2, max_gt=3, max_pr=4, seed=3)
    name = sorted(videos)[0]
    gt, pr = videos[name]
    frame = [f for f in gt['annolist'] if f['annorect']][0]
    frame['annorect'] = [dict(frame['annorect'][0], track_id=[k]) for k in range(65)]
    pack = E.PoseTrackPack(*E.load_data_dir(*_write(tmp_path / 'gt65', videos)))
    with pytest.raises(ValueError, match='65 GT people .at most 64'):
        E.evaluate_pack(pack)
    videos = S.make_videos(n_videos=1, frames=2, labelled=2, max_gt=3, max_pr=4, seed=3)
    gt, pr = videos[name]
    frame = [f for f in pr['annolist'] if f['annorect']][0]
    frame['annorect'] = frame['annorect'][:1] * 225
    pack = E.PoseTrackPack(*E.load_data_dir(*_write(tmp_path / 'pr225', videos)))
    with pytest.raises(ValueError, match='225 predicted people .at most 224'):
        E.evaluate_pack(pack)


def test_abi_rejects_bad_arguments_without_a_gpu():
    lib = L.lib()
    sz = C.c_size_t(0)
    cases = [
        ('dt_posetrack_assign', (None, None, None, 4, None, None, None, 65, 10, None, None, None, None), b'max_gt=65'),
        ('dt_posetrack_assign', (None, None, None, 4, None, None, None, 10, 225, None, None, None, None), b'max_pr=225'),
        ('dt_posetrack_assign', (None, None, None, 4, None, None, None, 10, 10, None, None, None, None), b'null pointer'),
        ('dt_posetrack_ap_workspace_bytes', (-1, C.byref(sz)), b'nentries=-1'),
        ('dt_posetrack_ap', (None, None, None, 4, None, None, None, 2, 100, None, None, 16, None), b'workspace of 16 B'),
        ('dt_posetrack_mot_smem_bytes', (10, 10, 5000, C.byref(sz)), b'map_cap=5000'),
        ('dt_posetrack_mot', (None,) * 10 + (3, 10, 300, 16, None, None, None, None), b'max_pr=300'),
        ('dt_posetrack_mot', (None,) * 10 + (3, 10, 10, 16, None, None, None, None), b'null pointer'),
    ]
    for name, args, msg in cases:
        rc = getattr(lib, name)(*args)
        assert rc != 0, name
        assert msg in lib.dt_last_error(), (name, lib.dt_last_error())


def test_size_queries_are_host_only():
    a, b = C.c_size_t(0), C.c_size_t(0)
    L.call('dt_posetrack_ap_workspace_bytes', 1000, C.byref(a))
    L.call('dt_posetrack_ap_workspace_bytes', 2000, C.byref(b))
    assert 0 < a.value < b.value
    L.call('dt_posetrack_mot_smem_bytes', 64, 224, 4096, C.byref(a))
    assert a.value <= 227 * 1024                                           # the worst case fits one SM
    L.call('dt_posetrack_mot_smem_bytes', 8, 12, 20, C.byref(b))
    assert b.value < a.value


def test_print_table_rows():
    header, row = E.print_table(Z['val3/apAll'])
    assert header == '& Head & Shou & Elb  & Wri  & Hip  & Knee & Ankl & Total\\\\\n'
    cum = E.get_cum(Z['val3/apAll'])
    assert len(cum) == 8 and cum[-1] == Z['val3/apAll'][-1, 0]
    assert row == E.get_format_row(cum) + '\n' and row.endswith(' \\\\\n')
    header, row = E.print_table(Z['val3/metrics'], motHeader=True)
    assert header.count('MOTA') == 8 and len(E.get_cum(Z['val3/metrics'])) == 11


def test_per_video_scores_file(tmp_path):
    from detectandtrack_b200.core import mpii_eval_engine as me
    path = str(tmp_path / 'scores.txt')
    paths = {'a/v1': '/x/v1.json', 'a/v2': '/x/v2.json', 'a/v3': '/x/v3.json'}
    me._write_per_video_scores(path, paths, {'v1.json': (np.float64(50.5), np.float64(10.0)),
                                             'v2.json': (np.nan, np.nan), 'v3.json': (np.float64(20.25), np.float64(-3.5))})
    rows = [('a/v1', np.float64(50.5), np.float64(10.0)), ('a/v2', np.nan, np.nan), ('a/v3', np.float64(20.25), np.float64(-3.5))]
    want = ''.join('{} {} {}\n'.format(*r) for r in sorted(rows, key=lambda x: x[1]))
    assert open(path).read() == want


def test_dataset_without_directories_takes_the_cfg_keys(tmp_path):
    """With EVAL.POSETRACK_ANNOTATION_DIR unset the JSON files are written and not scored; set, a dataset without its
    own annotation_directory is scored against it (here a directory that does not exist, so an IOError naming it)."""
    import pickle
    import types
    from detectandtrack_b200.core import config as Cfg
    from detectandtrack_b200.core import mpii_eval_engine as me
    Cfg.reset_cfg()
    assert Cfg.cfg.EVAL.POSETRACK_ANNOTATION_DIR == '' and Cfg.cfg.EVAL.POSETRACK_IMAGE_DIR == ''
    roidb = [{'image': 'images/v/%05d.jpg' % i, 'frame_id': i + 1} for i in range(2)]
    dets = {'all_boxes': [[], [np.zeros((0, 5), np.float32)] * 2], 'all_keyps': [[], [[], []]], 'all_tracks': [[], [[], []]]}
    with open(tmp_path / 'detections_withTracks.pkl', 'wb') as f:
        pickle.dump(dets, f)
    dataset = types.SimpleNamespace(name='posetrack_val')
    paths, res = me.run_mpii_eval(str(tmp_path), roidb, dataset)
    assert res is None and os.path.exists(paths['images/v'])
    Cfg.cfg.EVAL.POSETRACK_ANNOTATION_DIR = str(tmp_path / 'missing')
    try:
        with pytest.raises(IOError, match='missing'):
            me.run_mpii_eval(str(tmp_path), roidb, dataset)
    finally:
        Cfg.reset_cfg()
