"""Farneback flow between key frames on the device (csrc/flow.cu), with the reference's parameters (levels 10,
iterations 10, poly_n 7, poly_sigma 1.5, Gaussian window min(H, W) // 5), beside cv2's single-core time on the same pairs.

    python tools/bench_flow.py [--pairs 8] [--reps 5] [--cv2-pairs 1] [--out flow.json]

Per frame size (720x1280 and 1080x1920; a video of --pairs + 1 textured frames, every consecutive pair in one call):
  - pairs/s of dt_farneback_flow (CUDA events over --reps calls after a warm-up call) and of dt_flow_mean_abs;
  - the time of each kernel per call (torch.profiler, in a run of its own after the timed calls);
  - peak device memory per pair (frames, workspace and flows, from torch.cuda.max_memory_allocated);
  - cv2.calcOpticalFlowFarneback with cv2.setNumThreads(1) on --cv2-pairs of the same pairs, and the largest |d| of the
    device flow from it.
The card's name and power limit are read in the same call and printed with the numbers (one JSON line)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return dict(torch_name=torch.cuda.get_device_name(0), nvidia_smi=q[0] if q else 'unavailable')


def video(h, w, n, seed=0):
    """n BGR frames of low-passed noise drifting by about (1.5, -0.7) px per frame."""
    import cv2
    rng = np.random.RandomState(seed)
    base = cv2.GaussianBlur(rng.rand(h + 64, w + 64, 3).astype(np.float32), (0, 0), 3)
    base = ((base - base.min()) / (base.max() - base.min()) * 255).astype(np.float32)
    out = []
    for t in range(n):
        M = np.float32([[1, 0, 1.5 * t], [0, 1, -0.7 * t]])
        f = cv2.warpAffine(base, M, (w + 64, h + 64), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_REFLECT)
        out.append(np.clip(f[32:32 + h, 32:32 + w], 0, 255).astype(np.uint8))
    return np.stack(out)


def bench_size(h, w, args):
    import cv2
    import torch
    from detectandtrack_b200.ops import flow_ops
    frames = video(h, w, args.pairs + 1)
    pairs = [(i, i + 1) for i in range(args.pairs)]
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base_mem = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    d = torch.from_numpy(frames).cuda()
    flows = flow_ops.farneback_flow(d, pairs)                     # warm-up
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base_mem
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(args.reps):
        flows = flow_ops.farneback_flow(d, pairs)
    ev[1].record()
    torch.cuda.synchronize()
    ms = ev[0].elapsed_time(ev[1]) / args.reps
    ev[0].record()
    for _ in range(args.reps):
        flow_ops.flow_mean_abs(flows)
    ev[1].record()
    torch.cuda.synchronize()
    ms_mean = ev[0].elapsed_time(ev[1]) / args.reps
    # per-kernel times, one profiled call
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        flow_ops.farneback_flow(d, pairs)
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.key_averages():
        if e.device_type.name == 'CUDA' and getattr(e, 'device_time_total', 0) > 0:
            name = e.key.split('(')[0].split('<')[0].replace('dt::', '').replace('void ', '')
            kernels[name] = round(kernels.get(name, 0.0) + e.device_time_total / 1000.0, 3)
    # cv2 on one core, same pairs
    cv2.setNumThreads(1)
    gray = [cv2.cvtColor(f, cv2.COLOR_BGR2GRAY) for f in frames]
    fl = flows.cpu().numpy()
    t0 = time.time()
    err = 0.0
    for i in range(args.cv2_pairs):
        ref = cv2.calcOpticalFlowFarneback(gray[i], gray[i + 1], None, 0.5, 10, min(h, w) // 5, 10, 7, 1.5,
                                           cv2.OPTFLOW_FARNEBACK_GAUSSIAN)
        err = max(err, float(np.abs(ref - fl[i]).max()))
    cv2_s = (time.time() - t0) / args.cv2_pairs
    return dict(size='%dx%d' % (h, w), pairs=args.pairs, ms_per_call=round(ms, 3), pairs_per_s=round(args.pairs * 1000.0 / ms, 2),
                mean_abs_ms_per_call=round(ms_mean, 4), kernel_ms_per_call=kernels,
                peak_mb_per_pair=round(peak / args.pairs / 2 ** 20, 1), cv2_single_core_s_per_pair=round(cv2_s, 3),
                max_abs_diff_vs_cv2_px=err)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--pairs', type=int, default=8)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--cv2-pairs', type=int, default=1)
    ap.add_argument('--out', default='')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_flow needs a CUDA device')
    res = dict(card=card(), sizes=[bench_size(720, 1280, args), bench_size(1080, 1920, args)])
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
