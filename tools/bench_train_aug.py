#!/usr/bin/env python
"""The TRAIN.AUGMENT training step at BASELINE.json configs[4] size: 2 clips of T = 3 frames from 1280x720 sources,
R50-FPN-3D keypoint R-CNN, BATCH_SIZE_PER_IM 512, at the TRAIN.SCALES of configs/video/2d_best
(640 .. 800, MAX_SIZE 1333).  One JSON line with

  * step_ms per drawn scale (KeypointRcnnTrainer.step_clips, clip 1 flipped), next to step() at the default path;
  * dt_prep_batch against dt_prep_clip kernel time from torch.profiler (a run of its own);
  * peak torch.cuda.max_memory_allocated over 12 steps cycling all six scales against the 800-scale step: the blob and
    every activation shrink with the scale, so the cycle must stay within MEM_MARGIN of the 800-scale peak.

    python tools/bench_train_aug.py [--steps 10] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SCALES = (640, 672, 704, 736, 768, 800)
MEM_MARGIN = 64 << 20          # allocator rounding of the differently sized blocks of a smaller step


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    from bench import bench_cfg, synth_frames, synth_gt
    from detectandtrack_b200 import _lib as L
    from detectandtrack_b200.modeling import params as P
    from detectandtrack_b200.modeling.trainer import KeypointRcnnTrainer, pack_gt
    L.require_cuda()
    H, W, B, T = 720, 1280, 2, 3
    cfg = bench_cfg(800, 1333, 'r50fpn3d')
    cfg.TRAIN.BATCH_SIZE_PER_IM = 512; cfg.TRAIN.RPN_PRE_NMS_TOP_N = 2000
    cfg.TRAIN.SCALES, cfg.TRAIN.MAX_SIZE = SCALES, 1333
    blobs, spec = P.random_blobs(cfg)
    tr = KeypointRcnnTrainer(cfg, blobs, spec)
    frames = torch.from_numpy(synth_frames(B, T, H, W, 100)).cuda()
    clips = [frames[b].contiguous() for b in range(B)]
    gt = pack_gt(synth_gt(B, H, W, 7))
    flips = [0, 1]

    def timed(fn, n):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    res = dict(gpu=gpu_info(), workload='configs[4]: R50-FPN-3D keypoint R-CNN, %d clips x T=%d, %dx%d sources' % (B, T, W, H),
               step_ms_default=timed(lambda: tr.step(frames, gt), a.steps), step_ms_per_scale={})
    for s in SCALES:
        res['step_ms_per_scale'][s] = timed(lambda: tr.step_clips(clips, gt, [s, s], flips), a.steps)
    # peak memory: the 800-scale step, then 12 steps cycling the six scales
    torch.cuda.synchronize(); torch.cuda.reset_peak_memory_stats()
    for _ in range(3):
        tr.step_clips(clips, gt, [800, 800], flips)
    torch.cuda.synchronize()
    peak800 = torch.cuda.max_memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    for i in range(12):
        tr.step_clips(clips, gt, [SCALES[i % 6], SCALES[(i + 3) % 6]], flips)
    torch.cuda.synchronize()
    peak_cycle = torch.cuda.max_memory_allocated()
    res.update(peak_mib_800=peak800 / 2.0 ** 20, peak_mib_cycle=peak_cycle / 2.0 ** 20, mem_margin_mib=MEM_MARGIN / 2.0 ** 20,
               mem_ok=bool(peak_cycle <= peak800 + MEM_MARGIN))
    # kernel time of the two blob builders, in a profiled run of its own
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            tr.step(frames, gt)
            tr.step_clips(clips, gt, [800, 800], flips)
        torch.cuda.synchronize()
    kt = {}
    for ev in prof.key_averages():
        for k in ('prep_batch_kernel', 'prep_clip_kernel'):
            if k in ev.key:
                t = getattr(ev, 'device_time_total', None) or getattr(ev, 'cuda_time_total', 0)
                kt.setdefault(k, [0.0, 0])
                kt[k][0] += t; kt[k][1] += ev.count
    res['prep_kernel_us'] = {k: v[0] / max(1, v[1]) for k, v in kt.items()}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'bench_train_aug.json'), 'w') as f:
            f.write(line + '\n')
    return 0 if res['mem_ok'] else 1


if __name__ == '__main__':
    sys.exit(main())
