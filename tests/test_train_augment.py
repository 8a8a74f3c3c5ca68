"""CPU: the TRAIN.AUGMENT minibatch recipe on the host — flipped roidb entries, clip assembly over them, the per-clip scale
draw and blob geometry — against outputs of the REFERENCE's own functions (tests/golden/train_aug.npz,
tests/golden/gen_golden_train_aug.py); tools/train_net.py with a stub trainer; dt_prep_batch's argument checks."""
import ctypes as C
import importlib.util
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
G = np.load(os.path.join(HERE, 'golden', 'train_aug.npz'))
sys.path.insert(0, os.path.join(HERE, 'golden'))
sys.path.insert(0, HERE)


@pytest.mark.parametrize('tag,name', [('posetrack', 'posetrack_v1.0_train'), ('coco', 'keypoints_coco_2014_train')])
def test_flipped_entries_equal_reference(tag, name):
    from gen_golden_train_aug import frame_roidb
    from detectandtrack_b200.utils import roidb as R
    pairs = R.keypoint_flip_pairs(os.path.join('/data', name + '.json'))
    assert sorted(pairs) == [tuple(p) for p in G[tag + '_pairs'].tolist()]
    roidb = frame_roidb()
    n0 = len(roidb)
    orig = [dict(e) for e in roidb]
    R.extend_with_flipped_entries(roidb, pairs)
    assert len(roidb) == int(G[tag + '_n']) == 2 * n0
    for i, e in enumerate(roidb[n0:]):
        assert e['flipped'] is True and roidb[i]['flipped'] is False
        assert np.array_equal(e['boxes'], G['%s_%d_boxes' % (tag, i)]) and e['boxes'].dtype == G['%s_%d_boxes' % (tag, i)].dtype
        assert np.array_equal(e['gt_keypoints'], G['%s_%d_kps' % (tag, i)])
        assert e['image'] == orig[i]['image'] and e['width'] == orig[i]['width'] and e['frame_id'] == orig[i]['frame_id']
        assert np.array_equal(roidb[i]['boxes'], orig[i]['boxes'])          # the originals are untouched


def test_flip_boxes_of_tubes_equal_reference_per_frame():
    from detectandtrack_b200.utils.boxes import flip_boxes
    assert np.array_equal(flip_boxes(G['tubes_in'], int(G['tubes_width'])), G['tubes_flipped'])


def test_get_clip_over_flipped_entries_equals_reference():
    from gen_golden_train_aug import frame_roidb
    from detectandtrack_b200.core.config import cfg, reset_cfg
    from detectandtrack_b200.utils import roidb as R, video
    reset_cfg()
    try:
        cfg.VIDEO.NUM_FRAMES, cfg.VIDEO.NUM_FRAMES_MID, cfg.VIDEO.TIME_INTERVAL = 3, 1, 1
        roidb = R.extend_with_flipped_entries(frame_roidb(), R.keypoint_flip_pairs('posetrack_v1.0_train'))
        for e in roidb:
            e['gt_overlaps'] = np.tile(np.array([[0., 1.]], np.float32), (len(e['boxes']), 1))
        res = video.get_clip(roidb)
        assert len(res) == int(G['clip_n'])
        for i, e in enumerate(res):
            assert e['image'] == G['clip_%d_image' % i].tolist() and e['flipped'] == bool(G['clip_%d_flipped' % i])
            for k in ('tracks', 'boxes', 'gt_keypoints', 'track_visible'):
                assert np.array_equal(e[k], G['clip_%d_%s' % (i, k)]), (i, k)
    finally:
        reset_cfg()


def test_training_roidb_of_a_json_list_equals_reference(tmp_path):
    """utils/roidb.training_roidb on a JSON list of per-frame entries: the flipped copies are appended before clip assembly,
    so the clips equal the reference's get_clip over its flipped-extended roidb; without flip it is dataset.get_roidb."""
    import json
    from gen_golden_train_aug import frame_roidb
    from detectandtrack_b200.core import test_engine as te
    from detectandtrack_b200.core.config import cfg, reset_cfg
    from detectandtrack_b200.utils.roidb import training_roidb
    keep = ('image', 'frame_id', 'flipped', 'height', 'width', 'id', 'nframes', 'tracks', 'boxes', 'gt_keypoints', 'gt_classes', 'is_crowd')
    path = str(tmp_path / 'posetrack_frames.json')
    with open(path, 'w') as f:
        json.dump([{k: (v.tolist() if hasattr(v, 'tolist') else v) for k, v in e.items() if k in keep} for e in frame_roidb()], f)
    reset_cfg()
    try:
        cfg.MODEL.VIDEO_ON = True
        cfg.VIDEO.NUM_FRAMES, cfg.VIDEO.NUM_FRAMES_MID, cfg.VIDEO.TIME_INTERVAL = 3, 1, 1
        res = training_roidb(te.get_dataset(path), True)
        assert len(res) == int(G['clip_n'])
        for i, e in enumerate(res):
            assert e['image'] == G['clip_%d_image' % i].tolist() and e['flipped'] == bool(G['clip_%d_flipped' % i])
            for k in ('tracks', 'boxes', 'gt_keypoints', 'track_visible'):
                assert np.array_equal(e[k], G['clip_%d_%s' % (i, k)]), (i, k)
        plain = training_roidb(te.get_dataset(path), False)
        ref = te.get_dataset(path).get_roidb(gt=True)
        assert len(plain) == len(ref) == int(G['clip_n']) // 2
        assert [e['image'] for e in plain] == [e['image'] for e in ref] and not any(e.get('flipped') for e in plain)
    finally:
        reset_cfg()


def test_batch_geometry_equals_reference_blob():
    """Scale draw (stream 5 at counters 0, 1), prep_im_for_blob scale / resized size per clip, and the padded blob size
    equal _get_image_blob's; MAX_SIZE binds for the portrait clip."""
    from gen_golden_train_aug import BLOB_SCALES, BLOB_MAX_SIZE, SEED
    from detectandtrack_b200.modeling.engine import im_scale_and_size, padded_blob_size
    from detectandtrack_b200.ops.target_ops import train_scale
    targets = [train_scale(BLOB_SCALES, SEED, j) for j in range(2)]
    assert targets == G['blob_targets'].tolist()
    srcs = [G['blob_frames0'].shape[1:3], G['blob_frames1'].shape[1:3]]
    geo = [im_scale_and_size(h, w, t, BLOB_MAX_SIZE) for (h, w), t in zip(srcs, targets)]
    assert [s for s, _ in geo] == G['blob_im_scales'].tolist()
    assert [list(hw) for _, hw in geo] == G['blob_resized'].tolist()
    assert np.round(max(srcs[1]) * (targets[1] / float(min(srcs[1])))) > BLOB_MAX_SIZE     # MAX_SIZE binds for clip 1
    assert padded_blob_size([hw for _, hw in geo], 32.0) == tuple(G['blob'].shape[-2:])
    assert im_scale_and_size(96, 128, 96, 128) == (1.0, (96, 128))                             # the scale == 1.0 copy path


def test_scale_draw_equals_oracle_randint_on_stream_5():
    from oracle import targets as ot
    from detectandtrack_b200.ops.target_ops import hash_u32, train_scale
    scales = (640, 672, 704, 736, 768, 800)
    for seed in (3, 2 ** 40 + 7):
        ref = ot.randint(len(scales), 10000, seed, 5, 0)
        got = [scales.index(train_scale(scales, seed, n)) for n in range(10000)]
        assert got == ref.tolist()
        assert [hash_u32(seed, 5, 0, n) for n in (0, 9999)] == ot.hash_u32(seed, 5, 0, np.array([0, 9999])).tolist()
    assert set(ot.randint(len(scales), 10000, 3, 5, 0).tolist()) == set(range(6))


# ---------------------------------------------------------------------- tools/train_net.py with a stub trainer
def _train_net():
    spec = importlib.util.spec_from_file_location('train_net', os.path.join(ROOT, 'tools', 'train_net.py'))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def _run(tmp_path, monkeypatch, opts, world=1, rank=0, out='out'):
    """train_model() with the trainer replaced by a stub; returns the stub's calls."""
    import torch
    import torch.distributed as dist
    from detectandtrack_b200.core.config import cfg, cfg_from_file, cfg_from_list, assert_and_infer_cfg, reset_cfg
    from detectandtrack_b200.modeling import model_builder, trainer
    from test_gpu_tools import TRAIN_YAML
    tn = _train_net()
    calls = []

    class Stub(object):
        blobs0 = {'a_w': np.zeros((2, 2), np.float32)}
        totals = torch.tensor([10., 5.])

        def step(self, frames, gt):
            calls.append(('step', frames.numpy().copy(), gt))
            return torch.tensor([0.5, 0.1]), torch.tensor([0.2, 0.1, 3.0, 8.0])

        def step_clips(self, clips, gt, targets, flipped):
            calls.append(('step_clips', [c.numpy().copy() for c in clips], gt, list(targets), list(flipped)))
            return torch.tensor([0.5, 0.1]), torch.tensor([0.2, 0.1, 3.0, 8.0])

        def export_blobs(self, b):
            return dict(b)
    monkeypatch.setenv('RANK', str(rank))
    monkeypatch.setenv('WORLD_SIZE', str(world))
    monkeypatch.setattr(dist, 'init_process_group', lambda *a, **k: None)
    monkeypatch.setattr(dist, 'destroy_process_group', lambda *a, **k: None)
    monkeypatch.setattr(torch.cuda, 'set_device', lambda d: None)
    monkeypatch.setattr(torch.Tensor, 'cuda', lambda self, *a, **k: self)
    monkeypatch.setattr(model_builder, 'create', lambda *a, **k: Stub())
    monkeypatch.setattr(trainer, 'pack_gt', lambda gts, K=17: gts)
    reset_cfg()
    y = tmp_path / 'cfg.yaml'
    y.write_text(TRAIN_YAML)
    cfg_from_file(str(y))
    cfg_from_list(['OUTPUT_DIR', str(tmp_path / out), 'TRAIN.SNAPSHOT_ITERS', '20'] + opts)
    assert_and_infer_cfg()
    tn.train_model()
    return tn, calls


def _expected(tn, it, world, rank, B=2, K=17):
    """What train_net must hand the trainer at iteration it: entries of the flipped-extended synthetic roidb (2 clips + 2
    flipped copies) in the seeded order, their drawn scales, and the gt (flipped like the entry)."""
    from detectandtrack_b200.core.config import cfg
    from detectandtrack_b200.core import test_engine as te
    from detectandtrack_b200.ops.target_ops import train_scale
    from detectandtrack_b200.utils.boxes import flip_boxes
    from detectandtrack_b200.utils.roidb import flip_keypoints, DEFAULT_FLIP_PAIRS
    roidb = te.get_dataset(cfg.TRAIN.DATASET).get_roidb(gt=True)                 # the originals; then their flipped copies
    n0 = len(roidb)
    order = np.random.RandomState(cfg.RNG_SEED).permutation(2 * n0)
    out = []
    for j in range(B):
        n = it * world * B + rank * B + j
        i = order[n % len(order)]
        e = roidb[i % n0]
        g = tn._synthetic_gt(e, K)
        if i >= n0:
            g = dict(boxes=flip_boxes(g['boxes'], e['width']), gt_keypoints=flip_keypoints(g['gt_keypoints'], DEFAULT_FLIP_PAIRS, e['width']))
        out.append(dict(frames=np.stack(te.read_image_video(e)), flipped=bool(i >= n0), target=train_scale(cfg.TRAIN.SCALES, cfg.RNG_SEED, n),
                        gt=g))
    return out


def test_train_net_without_augment_calls_step_as_before(tmp_path, monkeypatch):
    from detectandtrack_b200.core import test_engine as te
    from detectandtrack_b200.core.config import cfg, reset_cfg
    try:
        tn, calls = _run(tmp_path, monkeypatch, ['SOLVER.MAX_ITER', '4'])
        assert [c[0] for c in calls] == ['step'] * 4
        roidb = te.get_dataset(cfg.TRAIN.DATASET).get_roidb(gt=True)
        order = np.random.RandomState(cfg.RNG_SEED).permutation(len(roidb))
        for it, (_, frames, gt) in enumerate(calls):
            entries = [roidb[order[(it * 2 + j) % len(order)]] for j in range(2)]
            assert frames.shape == (2, 3, 96, 128, 3) and frames.dtype == np.uint8
            assert np.array_equal(frames, np.stack([np.stack(te.read_image_video(e)) for e in entries]))
            for g, e in zip(gt, entries):
                ref = tn._synthetic_gt(e, 17)
                assert np.array_equal(g['boxes'], ref['boxes']) and np.array_equal(g['gt_keypoints'], ref['gt_keypoints'])
    finally:
        reset_cfg()


@pytest.mark.parametrize('world,rank', [(1, 0), (2, 0), (2, 1)])
def test_train_net_with_augment_draws_entries_flips_and_scales(tmp_path, monkeypatch, world, rank):
    from detectandtrack_b200.core.config import reset_cfg
    try:
        tn, calls = _run(tmp_path, monkeypatch, ['SOLVER.MAX_ITER', '12', 'TRAIN.AUGMENT', 'True', 'TRAIN.SCALES', '(64, 80, 96)'],
                         world=world, rank=rank)
        assert [c[0] for c in calls] == ['step_clips'] * 12
        seen_flip, seen_targets = set(), set()
        for it, (_, clips, gt, targets, flipped) in enumerate(calls):
            exp = _expected(tn, it, world, rank)
            assert flipped == [x['flipped'] for x in exp] and targets == [x['target'] for x in exp]
            for c, g, x in zip(clips, gt, exp):
                assert c.shape == (3, 96, 128, 3) and np.array_equal(c, x['frames'])         # unflipped: the device mirrors
                assert np.array_equal(g['boxes'], x['gt']['boxes']) and np.array_equal(g['gt_keypoints'], x['gt']['gt_keypoints'])
            seen_flip |= set(flipped)
            seen_targets |= set(targets)
        assert seen_flip == {False, True} and seen_targets == {64, 80, 96}
    finally:
        reset_cfg()


def test_train_net_with_augment_resumes_with_the_same_draws(tmp_path, monkeypatch):
    from detectandtrack_b200.core.config import cfg_from_list, reset_cfg
    try:
        opts = ['SOLVER.MAX_ITER', '45', 'TRAIN.AUGMENT', 'True', 'TRAIN.SCALES', '(64, 80, 96)']
        tn, calls = _run(tmp_path, monkeypatch, opts)
        assert len(calls) == 45
        d = os.path.join(str(tmp_path / 'out'), 'train', 'synthetic_1x2_96x128', 'keypoint_rcnn')
        os.remove(os.path.join(d, 'model_final.pkl'))                       # model_iter39.pkl is the newest: resume at 40
        _, again = _run(tmp_path, monkeypatch, opts + ['CLUSTER.ON_CLUSTER', 'True'])
        assert len(again) == 5
        for a, b in zip(calls[40:], again):
            assert a[3] == b[3] and a[4] == b[4]
            assert all(np.array_equal(x, y) for x, y in zip(a[1], b[1]))
    finally:
        reset_cfg()


# ---------------------------------------------------------------------- dt_prep_batch host checks (no GPU needed)
def _prep_batch_args(B=2, T=3, frames=(16, 32), H=(60, 90), W=(80, 50), scale=(1.2, 1.1), Hr=(72, 100), Wr=(96, 56),
                     Hp=128, Wp=96, Cp=8, row_planes=1, mode=0, null_arrays=False):
    ia = lambda v: (C.c_int * len(v))(*v)
    fr = (C.c_void_p * len(frames))(*frames)
    args = [fr, ia(H), ia(W), (C.c_double * len(scale))(*scale), ia(Hr), ia(Wr), ia([1, 0][:len(H)] + [0] * max(0, len(H) - 2)),
            B, T, (C.c_float * 3)(102.9801, 115.9465, 122.7717), Hp, Wp, Cp, 3, 4, row_planes, mode, C.c_void_p(64), None]
    if null_arrays:
        args[0] = None
    return args


@pytest.mark.parametrize('kw,msg', [
    (dict(B=0), b'1 <= B <= 16'),
    (dict(B=17), b'1 <= B <= 16'),
    (dict(T=0), b'T >= 1'),
    (dict(null_arrays=True), b'null pointer'),
    (dict(frames=(16, 0)), b'null frame pointer of clip 1'),
    (dict(H=(60, 0)), b'clip 1 has source size'),
    (dict(W=(0, 50)), b'clip 0 has source size'),
    (dict(scale=(1.2, 0.0)), b'clip 1 has im_scale'),
    (dict(Hr=(72, 129)), b'does not fit the padded'),
    (dict(Wr=(97, 56)), b'does not fit the padded'),
    (dict(Hp=127), b'row planes need an even padded height'),
    (dict(mode=3, Cp=16), b'bad output mode 3'),
    (dict(mode=4), b'bad output mode 4'),
    (dict(Cp=2, row_planes=0), b'bad output mode'),
], ids=lambda v: None if isinstance(v, dict) else v.decode()[:24].replace(' ', '_'))
def test_prep_batch_rejects_bad_arguments_without_a_gpu(kw, msg):
    from detectandtrack_b200 import _lib as L
    lib = L.lib()
    rc = lib.dt_prep_batch(*_prep_batch_args(**kw))
    err = lib.dt_last_error()
    assert rc != 0 and msg in err, err
    assert b'dt_prep_batch' in err
    with pytest.raises(RuntimeError, match='dt_prep_batch'):
        L.check(rc, 'dt_prep_batch')
    assert L.PREP_MAX_CLIPS == 16
