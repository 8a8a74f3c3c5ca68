"""Time one bf16x3 keypoint-head layer, direct against Winograd F(2x2, 3x3), at the benchmarked head size.

    python tools/bench_kps_head.py [--rois 832] [--reps 20]

Per repetition, in alternating order, each with L2 flushed first and CUDA events around the launches alone:
  direct        the 512 -> 512 3x3 conv as dt_conv3d (bf16x3, bias, ReLU, bf16-pair output)
  wino_gemm     dt_wino_gemm alone (16 products, K = 512 each)
  wino_xform    dt_wino_output_input alone (M + bias + ReLU -> pairs -> V of the next layer)
  wino_layer    dt_wino_gemm + dt_wino_output_input: what a middle head layer costs on the Winograd path
Prints the card, its power limit and one JSON line of median times (ms), achieved rates and wino_layer / direct.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                   # the numbers still print; the card line says why it is missing
        q = 'nvidia-smi unavailable (%s)' % e
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rois', type=int, default=832, help='RoIs of the head (8 clips x 104 detection slots)')
    ap.add_argument('--reps', type=int, default=20)
    args = ap.parse_args()
    import numpy as np
    import torch
    from detectandtrack_b200.ops import conv as cv
    D, S, C = args.rois, 14, 512
    G = D * (S // 2) ** 2
    rng = np.random.RandomState(0)
    w = (rng.randn(C, C, 3, 3) / np.sqrt(9 * C)).astype(np.float32)
    bias = torch.from_numpy((0.1 * rng.randn(C)).astype(np.float32)).cuda()
    wd = cv.pack_weight(torch.from_numpy(w), cv.BF16X3)
    wu = cv.pack_wino_weight(w)
    x = cv.split_bf16(torch.rand((D, 1, S, S, C), device='cuda'))
    y = torch.empty_like(x)
    v = torch.empty((16, G, 2 * C), dtype=torch.bfloat16, device='cuda')
    m = torch.empty((16, G, C), dtype=torch.float32, device='cuda')
    cv.wino_input(x, v)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')

    def direct():
        cv.conv3d(x, wd, (1, 3, 3), pad=(0, 1, 1), bias=bias, relu=True, dtype=cv.BF16X3, out=y, split_out=True, out_f32=False)

    def gemm():
        cv.wino_gemm(v, wu, m, G)

    def xform():
        cv.wino_output_input(m, D, S, C, bias, True, v)

    def layer():
        gemm()
        xform()
    runs = dict(direct=direct, wino_gemm=gemm, wino_xform=xform, wino_layer=layer)
    for f in runs.values():
        f()
    torch.cuda.synchronize()
    times = {k: [] for k in runs}
    for r in range(args.reps):
        order = list(runs) if r % 2 == 0 else list(runs)[::-1]
        for k in order:
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            runs[k]()
            e1.record()
            e1.synchronize()
            times[k].append(e0.elapsed_time(e1))
    med = {k: float(np.median(t)) for k, t in times.items()}
    # useful work: the direct conv's 9-tap products, the GEMM's 16 x K = 512 products, x3 for the split operands
    direct_flop = 2.0 * D * S * S * C * C * 9 * 3
    gemm_flop = 2.0 * 16 * G * C * C * 3
    xform_bytes = 16 * G * C * 4 + 16 * G * 2 * C * 2      # M read once, V written once
    print('card: %s' % card())
    print(json.dumps(dict(rois=D, reps=args.reps, ms=med, spread_ms={k: [min(t), max(t)] for k, t in times.items()},
                          direct_tflops=direct_flop / med['direct'] / 1e9, wino_gemm_tflops=gemm_flop / med['wino_gemm'] / 1e9,
                          wino_xform_tbps=xform_bytes / med['wino_xform'] / 1e9,
                          wino_layer_over_direct=med['wino_layer'] / med['direct'])))


if __name__ == '__main__':
    main()
