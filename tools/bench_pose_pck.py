"""The regular tracking pass with the 'pose-pck' cost on the device (TRACKING.DISTANCE_METRICS with a non-zero pose-pck
weight: dt_frame_costs + the batched solver + the id scan), next to the bbox-only pass of the same set as a control.

    python tools/bench_pose_pck.py [--reps 5] [--videos 64] [--out pose_pck.json]

The set is the tracking leg's shape: --videos videos of 30 frames with 100 detections each (the tracking leg's
generator, seed 3), a 17-joint pose per box on a quarter grid of the box plus jitter.  Per (weights, algo), the median of --reps
te._tracks_for_videos calls (host packing, the device passes and the copies back), host clock around synchronised work,
after one warm-up call.  One JSON line, with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WEIGHTS = {'bbox 1': (1.0, 0.0), 'bbox 1 + pose-pck 0.5': (1.0, 0.5), 'pose-pck 1': (0.0, 1.0)}


def card():
    import torch
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return dict(torch_name=torch.cuda.get_device_name(0), nvidia_smi=q[0] if q else 'unavailable')


def synth_video(rng, n_frames, n_dets):
    """The tracking leg's generator: random boxes in a 1333 x 800 frame, each frame the previous one jittered by
    N(0, 5^2) px with its rows permuted, scores U(0.95, 1), fp32."""
    x1 = rng.uniform(0, 1133, n_dets); y1 = rng.uniform(0, 500, n_dets)
    w = rng.uniform(30, 180, n_dets); h = rng.uniform(50, 300, n_dets)
    b = np.stack([x1, y1, x1 + w, y1 + h], 1)
    frames = []
    for f in range(n_frames):
        if f > 0:
            b = b + rng.normal(0, 5.0, b.shape)
            b = b[rng.permutation(n_dets)]
        frames.append(np.hstack([b, rng.uniform(0.95, 1.0, (n_dets, 1))]).astype(np.float32))
    return frames


def pose_set(videos, frames=30, dets=100, seed=3):
    rng = np.random.default_rng(seed)
    vb, vp = [], []
    for _ in range(videos):
        fr = synth_video(rng, frames, dets)
        ps = []
        for b in fr:
            g = rng.integers(0, 5, (2, b.shape[0], 17)) / 4.0
            x = b[:, 0:1] + g[0] * (b[:, 2:3] - b[:, 0:1]) + rng.normal(0, 2.0, (b.shape[0], 17))
            y = b[:, 1:2] + g[1] * (b[:, 3:4] - b[:, 1:2]) + rng.normal(0, 2.0, (b.shape[0], 17))
            p = np.stack([x, y, np.ones_like(x), np.ones_like(x)], 1).astype(np.float32)
            ps.append([p[i] for i in range(p.shape[0])])
        vb.append(fr); vp.append(ps)
    return vb, vp


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--videos', type=int, default=64)
    ap.add_argument('--out', default='')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_pose_pck needs a CUDA device')
    from detectandtrack_b200.core import tracking_engine as te
    from detectandtrack_b200.core.config import cfg, reset_cfg
    vb, vp = pose_set(args.videos)
    ms = {}
    for algo in ('hungarian', 'greedy'):
        for name, (wb, wp) in WEIGHTS.items():
            reset_cfg()
            cfg.TRACKING.DISTANCE_METRICS = ('bbox-overlap', 'pose-pck')
            cfg.TRACKING.DISTANCE_METRIC_WTS = (wb, wp)
            cfg.TRACKING.BIPARTITE_MATCHING_ALGO = algo
            te._tracks_for_videos(vb, vp)                                        # warm-up
            torch.cuda.synchronize()
            ts = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                te._tracks_for_videos(vb, vp)
                torch.cuda.synchronize()
                ts.append(time.perf_counter() - t0)
            ms['%s, %s' % (name, algo)] = round(1000 * sorted(ts)[len(ts) // 2], 2)
    reset_cfg()
    out = dict(card=card(), videos=args.videos, frames=30, detections=100, reps=args.reps, median_ms=ms)
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
