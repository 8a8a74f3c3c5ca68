"""The upper-bound experiments on the device: the tracking modes (TRACKING.DEBUG.UPPER_BOUND*, csrc/upper_bound.cu) at
the config-1 tracking scale, and poseval's upper-bound MOT (-u) on the PoseTrack-val-scale synthetic set.

    python tools/bench_upper_bound.py [--reps 5] [--oracle 1] [--out upper_bound.json]

Tracking: 10 videos of 30 frames, 100 detections per frame (oracle.tracking.synth_video's generator restated: jittered,
permuted boxes), each frame's GT the unjittered boxes with 17 integer keypoints; per mode, the time of --reps
compute_matches_tracks calls (host packing, the device passes and the copies back), host clock around synchronised work.
Evaluation: evaluate_pack with per-video scores on posetrack_synth.make_videos(seed=0), with and without
track_upper_bound, CUDA events around --reps evaluations.  Beside them, on one core, the CPU oracle
(tests/upper_bound_oracle.py, test infrastructure): the tracking modes with the bbox cost on the same set (the pose-pck
cost's per-pair Python loop would take hours), and the upper-bound MOT of the same loaded frames; --oracle 0 skips it.
One JSON line, with the card's name and power limit."""
import argparse
import copy
import importlib
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MODES = {'UPPER_BOUND': (1, 0, 0, 0), 'UPPER_BOUND_2_GT_KPS': (1, 1, 0, 0), 'UPPER_BOUND_5_GT_KPS_ONLY': (0, 0, 0, 1),
         'UPPER_BOUND + _5': (1, 0, 0, 1), 'none': (0, 0, 0, 0)}


def card():
    import torch
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return dict(torch_name=torch.cuda.get_device_name(0), nvidia_smi=q[0] if q else 'unavailable')


def tracking_set(n_videos=10, n_frames=30, n_dets=100, seed=0):
    rng = np.random.RandomState(seed)
    json_data, boxes, poses = [], [], []
    for v in range(n_videos):
        x1 = rng.uniform(0, 1133, n_dets); y1 = rng.uniform(0, 500, n_dets)
        b = np.stack([x1, y1, x1 + rng.uniform(30, 180, n_dets), y1 + rng.uniform(50, 300, n_dets)], 1)
        for f in range(n_frames):
            if f:
                b = b + rng.normal(0, 5.0, b.shape)
            kp = np.zeros((n_dets, 3, 17), np.int32)
            kp[:, 0] = np.round(rng.uniform(b[:, :1], b[:, 2:3], (n_dets, 17)))
            kp[:, 1] = np.round(rng.uniform(b[:, 1:2], b[:, 3:4], (n_dets, 17)))
            kp[:, 2] = 2
            json_data.append({'image': 'vid%03d/%05d.jpg' % (v, f), 'boxes': b.astype(np.float32), 'gt_keypoints': kp,
                              'tracks': np.arange(n_dets) + 1000 * v})
            perm = rng.permutation(n_dets)
            jb = b[perm] + rng.normal(0, 3.0, b.shape)
            boxes.append(np.hstack([jb, rng.uniform(0.95, 1.0, (n_dets, 1))]).astype(np.float32))
            p = np.zeros((n_dets, 4, 17), np.float32)
            p[:, :2] = kp[perm, :2] + rng.normal(0, 3.0, (n_dets, 2, 17))
            p[:, 2:] = rng.uniform(0, 1, (n_dets, 2, 17))
            poses.append(list(p))
    return json_data, boxes, poses


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--oracle', type=int, default=1)
    ap.add_argument('--out', default='')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_upper_bound needs a CUDA device')
    from detectandtrack_b200.core import tracking_engine as te
    from detectandtrack_b200.core.config import cfg, reset_cfg
    from detectandtrack_b200.datasets import posetrack_eval as E, posetrack_synth as S
    json_data, boxes, poses = tracking_set()
    track_ms = {}
    for w in (0.0, 1.0):
        for name, (ub, ub2, conf, ub5) in MODES.items():
            reset_cfg()
            d = cfg.TRACKING.DEBUG
            d.UPPER_BOUND, d.UPPER_BOUND_2_GT_KPS, d.UPPER_BOUND_2_GT_KPS_ONLY_CONF, d.UPPER_BOUND_5_GT_KPS_ONLY = \
                bool(ub), bool(ub2), bool(conf), bool(ub5)
            cfg.TRACKING.DISTANCE_METRICS = ('bbox-overlap', 'pose-pck')
            cfg.TRACKING.DISTANCE_METRIC_WTS = (1.0, w)
            mk = lambda: {'all_boxes': [[], [b.copy() for b in boxes]], 'all_keyps': [[], [[p.copy() for p in ps] for ps in poses]]}
            te.compute_matches_tracks(json_data, mk())                               # warm-up
            torch.cuda.synchronize()
            t = 0.0
            for _ in range(args.reps):
                dets = mk()
                t0 = time.perf_counter()
                te.compute_matches_tracks(json_data, dets)
                torch.cuda.synchronize()
                t += time.perf_counter() - t0
            track_ms['%s, pose-pck %g' % (name, w)] = round(1000 * t / args.reps, 2)
    reset_cfg()
    with tempfile.TemporaryDirectory() as tmp:
        gt_dir, pred_dir = S.write_dirs(S.make_videos(seed=0), tmp)
        gt, pr, names = E.load_data_dir(gt_dir, pred_dir)
    pack = E.PoseTrackPack(gt, pr, names)
    eval_ms = {}
    for ub in (False, True, False, True):
        E.evaluate_pack(pack, True, True, per_video=True, track_upper_bound=ub)      # warm-up
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        torch.cuda.synchronize()
        ev[0].record()
        for _ in range(args.reps):
            res = E.evaluate_pack(pack, True, True, per_video=True, track_upper_bound=ub)
        ev[1].record()
        torch.cuda.synchronize()
        eval_ms.setdefault('upper_bound' if ub else 'normal', []).append(round(ev[0].elapsed_time(ev[1]) / args.reps, 3))
        eval_ms['MOTA_upper_bound' if ub else 'MOTA'] = float(res['metrics'][-4, 0])
    out = dict(card=card(), tracking_frames=len(json_data), detections_per_frame=len(boxes[0]), tracking_ms=track_ms,
               eval_frames=pack.nframes, eval_ms=eval_ms)
    if args.oracle:
        os.environ.setdefault('OMP_NUM_THREADS', '1')
        sys.path.insert(0, os.path.join(ROOT, 'tests'))
        U = importlib.import_module('upper_bound_oracle')
        videos = {}
        for i, e in enumerate(json_data):
            videos.setdefault(os.path.dirname(e['image']), []).append(dict(
                boxes=boxes[i], poses=poses[i], gt_boxes=e['boxes'], gt_kps=e['gt_keypoints'], gt_tracks=e['tracks']))
        oracle_ms = {}
        for name, (ub, ub2, conf, ub5) in MODES.items():
            if name == 'none':
                continue
            t0 = time.perf_counter()
            for frames in videos.values():
                U.compute_tracks_video(frames, bool(ub), bool(ub2), bool(conf), bool(ub5), 1.0, 0.0, 'hungarian')
            oracle_ms['%s, pose-pck 0' % name] = round(1000 * (time.perf_counter() - t0), 2)
        t0 = time.perf_counter()
        metrics, _ = U.evaluate_tracking_upper_bound(copy.deepcopy(gt), copy.deepcopy(pr))
        out['oracle_tracking_ms'] = oracle_ms
        out['oracle_eval_upper_bound_ms'] = round(1000 * (time.perf_counter() - t0), 1)
        assert abs(float(metrics[-4, 0]) - eval_ms['MOTA_upper_bound']) <= 1e-12 * abs(eval_ms['MOTA_upper_bound'])
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
