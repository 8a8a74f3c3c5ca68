"""GPU: the TRAIN.AUGMENT minibatch on the device — dt_prep_batch against dt_prep_clip (byte for byte, flipped and ragged
batches included) and against the reference's _get_image_blob (tests/golden/train_aug.npz), the target generators at
per-clip im_info rows, KeypointRcnnTrainer.step_clips (flip equivalence, autograd of the oracle graph) and
tools/train_net.py end to end on a JSON roidb of mixed frame sizes."""
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import targets as ot

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
G = np.load(os.path.join(HERE, 'golden', 'train_aug.npz'))
MEANS = (102.9801, 115.9465, 122.7717)


def _unplane(x, row_planes):
    """[F, 2, Ht/2, Wt, C] (rows de-interleaved by parity) -> [F, Ht, Wt, C]."""
    if not row_planes:
        return x
    F, _, h2, Wt, Cc = x.shape
    full = np.empty((F, 2 * h2, Wt, Cc), x.dtype)
    full[:, 0::2], full[:, 1::2] = x[:, 0], x[:, 1]
    return full


# mode -> (cpad, border, row_planes): the engine's layouts (bf16 / bf16x3 conv1 blob, tf32 blob, raw fp32 blob)
MODES = {0: (8, (3, 4), True), 1: (4, (0, 0), False), 2: (4, (0, 0), False), 3: (8, (3, 4), True)}


@pytest.mark.parametrize('mode', [0, 1, 2, 3])
@pytest.mark.parametrize('flip', [0, 1])
def test_prep_batch_equals_prep_clip_per_clip(mode, flip):
    """A ragged batch (three source sizes; scale 1.0, an up-scale, a down-scale; the second clip flipped when flip) equals
    prep_clip of each clip alone (of the mirrored frames where flipped), byte for byte; everything outside each clip's
    Hr x Wr is zero."""
    import torch
    from detectandtrack_b200.ops import dense_ops
    rng = np.random.default_rng(11 + mode)
    T = 3
    srcs = [(45, 61), (45, 61), (70, 50)]
    scales = [1.0, 1.6, 0.53]
    sizes = [(45, 61), (72, 98), (37, 27)]
    flips = [0, flip, 0]
    frames = [rng.integers(0, 256, (T, h, w, 3), dtype=np.uint8) for h, w in srcs]
    Hp, Wp = 96, 128
    cpad, border, planes = MODES[mode]
    out = dense_ops.prep_batch([torch.from_numpy(f).cuda() for f in frames], MEANS, scales, sizes, flips, (Hp, Wp), cpad=cpad,
                               out_f32=mode, border=border, row_planes=planes)
    out = out.cpu()
    by, bx = border
    for b in range(3):
        src = np.ascontiguousarray(np.flip(frames[b], 2)) if flips[b] else frames[b]
        ref = dense_ops.prep_clip(torch.from_numpy(src).cuda(), MEANS, scales[b], sizes[b], (Hp, Wp), cpad=cpad, out_f32=mode,
                                  border=border, row_planes=planes).cpu()
        got = out[b * T:(b + 1) * T]
        assert got.shape == ref.shape
        assert torch.equal(got.contiguous().view(torch.uint8), ref.contiguous().view(torch.uint8)), (b, mode, flip)
        full = _unplane(got.float().numpy(), planes)
        hr, wr = sizes[b]
        inside = np.zeros(full.shape[1:3], bool)
        inside[by:by + hr, bx:bx + wr] = True
        assert np.all(full[:, ~inside] == 0) and np.all(full[..., 6:] == 0)
        assert np.abs(full[:, inside, :3]).max() > 0
    if flip:         # the flip is of the source, not of the resized image (cv2 maps columns through 1/fx)
        plain = dense_ops.prep_clip(torch.from_numpy(frames[1]).cuda(), MEANS, scales[1], sizes[1], (Hp, Wp), cpad=cpad,
                                    out_f32=mode, border=border, row_planes=planes).float().cpu().numpy()
        mirrored = _unplane(plain, planes)[:, by:by + 72, bx:bx + 98][:, :, ::-1]
        assert not np.array_equal(_unplane(out[T:2 * T].float().numpy(), planes)[:, by:by + 72, bx:bx + 98], mirrored)


def test_prep_batch_equals_reference_image_blob():
    """The reference's _get_image_blob (two clips, T = 2, landscape flipped + portrait with MAX_SIZE binding) against the
    raw fp32 blob, within test_prep_clip_resize_vs_cv2's tolerance; the padding is exactly zero."""
    import torch
    from detectandtrack_b200.ops import dense_ops
    frames = [G['blob_frames0'], G['blob_frames1']]
    blob = G['blob']                                                           # [B, 3, T, Hp, Wp]
    B, _, T, Hp, Wp = blob.shape
    sizes = [tuple(s) for s in G['blob_resized'].tolist()]
    out = dense_ops.prep_batch([torch.from_numpy(f).cuda() for f in frames], MEANS, G['blob_im_scales'].tolist(), sizes, [1, 0],
                               (Hp, Wp), cpad=4, out_f32=2).cpu().numpy()
    ref = blob.transpose(0, 2, 3, 4, 1).reshape(B * T, Hp, Wp, 3)
    np.testing.assert_allclose(out[..., :3], ref, rtol=1e-3, atol=2e-3)
    for b, (hr, wr) in enumerate(sizes):
        o = out[b * T:(b + 1) * T]
        assert np.all(o[:, hr:] == 0) and np.all(o[:, :, wr:] == 0) and np.all(o[..., 3] == 0)


def test_targets_at_per_clip_im_info_rows_equal_oracle():
    """A two-scale minibatch: each image's RPN targets and sampled RoIs equal the oracle at that image's own im_info row."""
    import torch
    from detectandtrack_b200.ops import target_ops
    from test_gpu_targets import _TrainCfg, _Cfg, _gt_tensors, _cmp_box_targets, _check_sampled, _anchors
    rng = np.random.default_rng(17)
    B, Gmax = 2, 8
    info = np.array([[72, 96, 1.2], [100, 56, 1.1111111111111112]], np.float32)
    shapes = [(int(np.ceil(128 / 2. ** l)), int(np.ceil(96 / 2. ** l))) for l in range(2, 7)]
    counts = np.array([3, 2], np.int32)
    boxes = np.zeros((B, Gmax, 4), np.float32)
    gts, kps = [], []
    for b in range(B):
        H, W = info[b, 0] / info[b, 2], info[b, 1] / info[b, 2]
        x1 = rng.uniform(0, W - 25, counts[b]); y1 = rng.uniform(0, H - 25, counts[b])
        g = np.stack([x1, y1, x1 + rng.uniform(8, 24, counts[b]), y1 + rng.uniform(8, 24, counts[b])], 1).astype(np.float32)
        boxes[b, :counts[b]] = g
        k = np.zeros((counts[b], 3, 17), np.int32)
        for i in range(counts[b]):
            k[i, 0] = rng.integers(int(g[i, 0]), int(g[i, 2]) + 1, 17); k[i, 1] = rng.integers(int(g[i, 1]), int(g[i, 3]) + 1, 17)
            k[i, 2] = rng.integers(0, 3, 17)
        gts.append(g); kps.append(k)
    im = torch.from_numpy(info).cuda()
    out = target_ops.rpn_targets(shapes, _anchors(torch), [2. ** l for l in range(2, 7)], 3, torch.from_numpy(boxes).cuda(),
                                 torch.from_numpy(counts).cuda(), im, _TrainCfg(64), 13)
    for b in range(B):
        lv = [(G_anchor, 2. ** lvl, H, W) for lvl, (H, W), G_anchor in zip(range(2, 7), shapes, [a.cpu().numpy() for a in _anchors(torch)])]
        ref, _ = ot.rpn_targets(lv, boxes[b, :counts[b]] * info[b, 2], float(info[b, 0]), float(info[b, 1]), 13, b, batch=64)
        for l, o in enumerate(out):
            assert np.array_equal(o['labels'][b].cpu().numpy(), ref[l]['labels']), (b, l)
            _cmp_box_targets(o['bbox_targets'][b].cpu().numpy(), ref[l]['bbox_targets'], 'img %d level %d' % (b, l))
            assert np.array_equal(o['inside'][b].cpu().numpy(), ref[l]['inside'])
            assert np.array_equal(o['outside'][b].cpu().numpy(), ref[l]['outside'])
    # RoI sampling: proposals in each image's blob coordinates
    R, topn, batch = 120, 200, 64
    rois, scores, cnts = [], [], []
    for b in range(B):
        n = 90 + 10 * b
        src = gts[b][rng.integers(0, counts[b], n)] + rng.normal(0, 3, (n, 4)).astype(np.float32)
        src[:, 2:] = np.maximum(src[:, 2:], src[:, :2] + 1)
        r = np.zeros((R, 5), np.float32); r[:, 0] = b; r[:n, 1:] = src * info[b, 2]
        sc = np.zeros((R,), np.float32); sc[:n] = np.sort(rng.uniform(0, 1, n).astype(np.float32))[::-1]
        rois.append(r); scores.append(sc); cnts.append(n)
    gt = _gt_tensors(torch, gts, [np.ones(len(g), np.int32) for g in gts], [np.zeros(len(g), np.int32) for g in gts], kps)
    o = target_ops.sample_rois(torch.from_numpy(np.stack(rois)).cuda(), torch.from_numpy(np.stack(scores)).cuda(),
                               torch.tensor(cnts, dtype=torch.int32).cuda(), gt, im, _Cfg(batch, topn), 21)
    kept = ot.collect_train([rois[b][:cnts[b]] for b in range(B)], [scores[b][:cnts[b]] for b in range(B)], topn)
    for b in range(B):
        ref = ot.sample_rois(gts[b], np.ones(len(gts[b]), np.int32), np.zeros(len(gts[b]), np.int32), kps[b], kept[b][:, 1:],
                             info[b, 2], b, 21, batch=batch)
        _check_sampled(o, b, ref, batch)


def _trainer_cfg():
    from test_gpu_engine import _cfg
    cfg = _cfg()
    cfg.TEST.SCALES = (96,); cfg.TEST.MAX_SIZE = 128
    cfg.TRAIN.MAX_SIZE = 128
    cfg.TRAIN.BATCH_SIZE_PER_IM = 64; cfg.TRAIN.RPN_PRE_NMS_TOP_N = 300; cfg.TRAIN.RPN_POST_NMS_TOP_N = 200
    cfg.TRAIN.RPN_BATCH_SIZE_PER_IM = 64
    return cfg


def _entries(rng, sizes, K=17):
    out = []
    for b, (H, W) in enumerate(sizes):
        g = 2 + b
        x1 = rng.uniform(0, W - 50, g); y1 = rng.uniform(0, H - 45, g)
        boxes = np.stack([x1, y1, x1 + rng.uniform(25, 48, g), y1 + rng.uniform(25, 43, g)], 1).astype(np.float32)
        kps = np.zeros((g, 3, K), np.int32)
        for i in range(g):
            kps[i, 0] = rng.randint(int(boxes[i, 0]), int(boxes[i, 2]) + 1, K)
            kps[i, 1] = rng.randint(int(boxes[i, 1]), int(boxes[i, 3]) + 1, K)
            kps[i, 2] = rng.randint(0, 3, K)
        out.append(dict(boxes=boxes, gt_keypoints=kps))
    return out


def test_step_clips_flip_on_the_device_equals_host_mirrored_frames():
    """step_clips with flipped=[1, 0] (the device mirrors clip 0) and the host-flipped gt, against step_clips on host-mirrored
    frames with flipped=[0, 0] and the same gt: the blob, RPN outputs and targets are bit-identical and the losses agree to
    1e-6 (the split-K gradient reduction is not bit-deterministic)."""
    import torch
    from detectandtrack_b200.modeling import params as P
    from detectandtrack_b200.modeling.trainer import KeypointRcnnTrainer, pack_gt
    from detectandtrack_b200.utils.roidb import flipped_entry, DEFAULT_FLIP_PAIRS
    cfg = _trainer_cfg()
    try:
        blobs, spec = P.random_blobs(cfg, seed=3)
        rng = np.random.RandomState(2)
        sizes = [(80, 120), (96, 72)]
        frames = [rng.randint(0, 256, (3, h, w, 3)).astype(np.uint8) for h, w in sizes]
        ents = _entries(rng, sizes)
        ents[0] = flipped_entry(dict(ents[0], width=sizes[0][1]), DEFAULT_FLIP_PAIRS)
        gt = pack_gt([dict(boxes=e['boxes'], gt_keypoints=e['gt_keypoints']) for e in ents])
        targets = [96, 64]
        runs = []
        for clips, flips in (([frames[0], frames[1]], [1, 0]), ([np.ascontiguousarray(frames[0][:, :, ::-1]), frames[1]], [0, 0])):
            tr = KeypointRcnnTrainer(cfg, blobs, spec, lr=0.01, weight_decay=1e-4)
            dev = [torch.from_numpy(c).cuda() for c in clips]
            x, hp, wp, im = tr.blob_clips(dev, targets, flips)
            outs = tr.forward_blob(x, 2, 3, hp, wp)
            r = dict(x=x.clone(), im=im.cpu(), outs=[o.clone() for o in outs])
            l1, l2 = tr.step_clips(dev, gt, targets, flips, seed=5)
            r.update(loss=torch.cat([l1, l2[:3]]).cpu().numpy(), rt=tr.last['rpn_targets'], smp=tr.last['sampled'])
            runs.append(r)
            del tr
        a, b = runs
        assert torch.equal(a['x'].view(torch.int16), b['x'].view(torch.int16)) and torch.equal(a['im'], b['im'])
        assert a['im'][:, :2].tolist() == [[85., 128.], [85., 64.]]                  # TRAIN.MAX_SIZE binds for clip 0
        for oa, ob in zip(a['outs'], b['outs']):
            assert torch.equal(oa, ob)
        for ta, tb in zip(a['rt'], b['rt']):
            for k in ta:
                assert torch.equal(ta[k], tb[k]), k
        for k in a['smp']:
            assert torch.equal(a['smp'][k], b['smp'][k]), k
        np.testing.assert_allclose(a['loss'], b['loss'], rtol=1e-6, atol=0)
        assert np.all(np.isfinite(a['loss']))
    finally:
        _trainer_cfg()


def test_step_clips_mixed_scale_vs_autograd():
    """A two-scale minibatch of a landscape and a portrait clip (one flipped, padded to the union of their sizes) through
    step_clips' pieces, against autograd of the oracle graph on the blob the device read, with
    test_keypoint_rcnn_training_step_vs_autograd's tolerances.  One exception: res3_0_branch2a, the first trainable layer
    and the end of the longest bf16 backward chain, gets cosine >= 0.975.  Measured here: 0.979 / 0.981 (this layout / two
    landscape clips), max-norm error 0.20 / 0.23, while every loss agrees to 0.3 % and every other checked layer has
    cosine >= 0.989."""
    import torch
    from detectandtrack_b200 import _lib as L_
    from detectandtrack_b200.modeling import params as P
    from detectandtrack_b200.modeling.trainer import KeypointRcnnTrainer, pack_gt
    from test_gpu_trainer import _oracle_full_step
    cfg = _trainer_cfg()
    try:
        blobs, spec = P.random_blobs(cfg, seed=3)
        rng = np.random.RandomState(0)
        sizes = [(96, 128), (120, 90)]
        frames = [rng.randint(0, 256, (3, h, w, 3)).astype(np.uint8) for h, w in sizes]
        gt = pack_gt(_entries(rng, sizes))
        tr = KeypointRcnnTrainer(cfg, blobs, spec, lr=0.01, weight_decay=1e-4)
        dev = [torch.from_numpy(f).cuda() for f in frames]
        targets, flips = [80, 96], [0, 1]
        x, hp, wp, im = tr.blob_clips(dev, targets, flips)
        assert im[:, 2].tolist() != [im[0, 2].item()] * 2                     # two scales
        outs = tr.forward_blob(x, 2, 3, hp, wp)
        rt, smp = tr.targets_at(outs, gt, im, 5)
        tr.forward_heads(smp)
        L_.call('dt_memset', L_.ptr(tr.flat_g), 0, tr.flat_g.numel() * 4, L_.stream_ptr())
        tr.reducer.reset()
        hg = tr.backward_heads(smp)
        loss = tr.backward(outs, rt, head_grads=hg, fresh=False).cpu().numpy()
        lh = tr.loss_heads.cpu().numpy()
        assert int(smp['counts'].min()) > 8 and int(smp['kp_counts'].sum()) > 0
        # the oracle's input: exactly the blob the device's conv1 read (bf16, de-interleaved rows, zero border cropped),
        # + means so the oracle's own mean subtraction gives it back
        xb = x.float().cpu().numpy()                                          # [B, T, 2, (hp + 6) / 2, wp + 8, Cp]
        full = np.empty(xb.shape[:2] + (2 * xb.shape[3],) + xb.shape[4:], np.float32)
        full[:, :, 0::2], full[:, :, 1::2] = xb[:, :, 0], xb[:, :, 1]
        data = full[:, :, 3:3 + hp, 4:4 + wp, :3]
        frames_f = data + np.asarray(cfg.PIXEL_MEANS, np.float32).reshape(1, 1, 1, 1, 3)
        rt_np = [{k: v.cpu().numpy() for k, v in t.items()} for t in rt]
        smp_np = {k: v.cpu().numpy() for k, v in smp.items()}
        ref_l, grads = _oracle_full_step(cfg, blobs, frames_f, rt_np, smp_np)
        got_l = [loss[0], loss[1], lh[0], lh[1], lh[2]]
        for name, a, b in zip(('rpn_cls', 'rpn_bbox', 'cls', 'bbox', 'kps'), got_l, ref_l):
            assert abs(a - b) <= 3e-2 * abs(b) + 1e-6, (name, a, b)

        def dev_grad(c):
            kT, kH, kW = c.k
            return c.g.view(kT, kH, kW, c.cout, c.cin).permute(3, 4, 0, 1, 2).cpu()
        bad = []

        def check(name, got, ref, tol=0.25, min_cos=0.985):
            ref = ref.reshape(got.shape)
            if float(ref.abs().max()) == 0.0 and float(got.abs().max()) == 0.0:
                return
            err = (got - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)
            cos = float((got.flatten() * ref.flatten()).sum() / (got.norm() * ref.norm() + 1e-30))
            errs[name] = (round(err, 4), round(cos, 5))
            if err > tol or cos < min_cos:
                bad.append((name, round(err, 4), round(cos, 5)))
        errs = {}
        g6 = dev_grad(tr.fc6)[:, :, 0, 0, 0].view(-1, 7, 7, 256).permute(0, 3, 1, 2).reshape(-1, 12544)
        check('fc6_w', g6, grads['fc6_w'])
        check('fc7_w', dev_grad(tr.fc7)[:, :, 0, 0, 0], grads['fc7_w'])
        for i in (0, 7):
            check('conv_fcn%d_w' % (i + 1), dev_grad(tr.kps[i])[:, :, 0], grads['conv_fcn%d_w' % (i + 1)])
        for i, n in enumerate(spec.stage_blobs[::-1]):
            check('fpn_' + n, dev_grad(tr.post[i]), grads['fpn_%s_w' % n])
        check('conv_rpn', dev_grad(tr.rpn_conv), grads['conv_rpn_fpn2_w'])
        check('res5_2_branch2c', dev_grad(tr.stages[-1][-1]['c']), grads['res5_2_branch2c_w'])
        check('res3_0_branch2a', dev_grad(tr.stages[0][0]['a']), grads['res3_0_branch2a_w'], min_cos=0.975)
        print('losses (device, oracle)', list(zip(got_l, ref_l)))
        print('grad (max-norm rel err, cosine) per layer', errs)
        assert not bad, bad
    finally:
        _trainer_cfg()


def test_train_net_augment_end_to_end_on_mixed_frame_sizes(tmp_path):
    """tools/train_net.py with TRAIN.AUGMENT on a JSON roidb of one landscape and one portrait video (jpgs written here):
    it runs, logs finite losses, and tools/test_net.py loads its model_final.pkl."""
    import re
    import cv2
    from test_gpu_tools import TRAIN_YAML
    rng = np.random.RandomState(4)
    entries = []
    for v, (H, W) in (('land', (96, 128)), ('port', (128, 96))):
        os.makedirs(str(tmp_path / v))
        for f in range(1, 4):
            path = str(tmp_path / v / ('%06d.jpg' % f))
            cv2.imwrite(path, rng.randint(0, 256, (H, W, 3)).astype(np.uint8))
            g = 2
            x1 = rng.uniform(0, W - 40, g); y1 = rng.uniform(0, H - 40, g)
            boxes = np.stack([x1, y1, x1 + 30, y1 + 35], 1)
            kps = np.zeros((g, 3, 17), np.int64)
            for i in range(g):
                kps[i, 0] = rng.randint(int(x1[i]), int(x1[i]) + 30, 17); kps[i, 1] = rng.randint(int(y1[i]), int(y1[i]) + 35, 17)
                kps[i, 2] = rng.randint(0, 3, 17)
            entries.append(dict(image=path, frame_id=f, height=H, width=W, boxes=boxes.tolist(), gt_keypoints=kps.tolist(),
                                tracks=[[0], [1]], gt_classes=[1, 1], is_crowd=[False, False]))
    roidb = str(tmp_path / 'posetrack_mixed.json')
    with open(roidb, 'w') as f:
        json.dump(entries, f)
    cfg = tmp_path / 'cfg.yaml'
    cfg.write_text(TRAIN_YAML)
    env = dict(os.environ, PYTHONPATH=ROOT)
    out = str(tmp_path / 'out')
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'train_net.py'), '--cfg', str(cfg), 'OUTPUT_DIR', out,
                        'TRAIN.DATASET', roidb, 'TRAIN.AUGMENT', 'True', 'TRAIN.SCALES', '(64, 80, 96)', 'TRAIN.MAX_SIZE', '128',
                        'SOLVER.MAX_ITER', '8'], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    losses = [float(m.group(1)) for m in re.finditer(r'iter \d+ lr [\d.]+ loss ([\d.]+)', r.stdout)]
    assert len(losses) == 2 and all(np.isfinite(losses)), r.stdout[-2000:]
    snap = os.path.join(out, 'train', 'posetrack_mixed', 'keypoint_rcnn', 'model_final.pkl')
    w = pickle.load(open(snap, 'rb'))
    assert w['blobs']['fc6_w'].shape == (1024, 12544)
    r2 = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'test_net.py'), '--cfg', str(cfg), 'OUTPUT_DIR', str(tmp_path / 'out2'),
                         'TEST.WEIGHTS', snap], env=env, capture_output=True, text=True, timeout=600)
    assert r2.returncode == 0, r2.stdout[-2000:] + r2.stderr[-2000:]
