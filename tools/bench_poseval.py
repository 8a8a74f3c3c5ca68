"""The device PoseTrack evaluation (csrc/poseval.cu) on a PoseTrack-val-scale synthetic set, beside the CPU oracle.

    python tools/bench_poseval.py [--reps 5] [--oracle 1] [--out poseval.json]

The set is posetrack_synth.make_videos() (seed 0): 50 videos of 118 frames, 53 labelled, up to 36 GT and 60 predictions
per frame, with per-video scores on (EVAL.EVAL_MPII_PER_VIDEO).  Reported (one JSON line):
  - device_ms: CUDA events around --reps complete device evaluations of the loaded pack (upload, the three launches,
    the copies back and the per-joint host arithmetic), after a warm-up evaluation, synchronised at both ends;
  - kernel_ms: the time of each kernel in one evaluation (torch.profiler, a run of its own after the timed ones);
  - host_load_s: reading the JSON files and packing them (the same for every evaluator);
  - oracle_s: the numpy/scipy oracle (oracle/poseval.py, test infrastructure) on one core on the same loaded frames,
    the dataset-level evaluation only (per-video scores would re-run it once per video), --oracle 0 to skip it;
  - the card's name and power limit, read in the same run."""
import argparse
import copy
import importlib
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return dict(torch_name=torch.cuda.get_device_name(0), nvidia_smi=q[0] if q else 'unavailable')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--oracle', type=int, default=1)
    ap.add_argument('--out', default='')
    args = ap.parse_args()
    os.environ.setdefault('OMP_NUM_THREADS', '1')
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_poseval needs a CUDA device')
    from detectandtrack_b200.datasets import posetrack_eval as E, posetrack_synth as S
    with tempfile.TemporaryDirectory() as tmp:
        gt_dir, pred_dir = S.write_dirs(S.make_videos(seed=0), tmp)
        t0 = time.time()
        gt, pr, names = E.load_data_dir(gt_dir, pred_dir)
        pack = E.PoseTrackPack(gt, pr, names)
        host_load = time.time() - t0
    res = E.evaluate_pack(pack, True, True, per_video=True)                          # warm-up
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(args.reps):
        res = E.evaluate_pack(pack, True, True, per_video=True)
    ev[1].record()
    torch.cuda.synchronize()
    ms = ev[0].elapsed_time(ev[1]) / args.reps
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        E.evaluate_pack(pack, True, True, per_video=True)
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.key_averages():
        if e.device_type.name == 'CUDA' and getattr(e, 'device_time_total', 0) > 0 and 'pt_' in e.key:
            name = e.key.split('(')[0].split('<')[0].replace('dt::', '').replace('void ', '')
            kernels[name] = round(kernels.get(name, 0.0) + e.device_time_total / 1000.0, 3)
    out = dict(card=card(), frames=pack.nframes, gt_people=int(pack.gt_off[-1]), predictions=int(pack.pr_off[-1]),
               sequences=len(pack.seq_ranges()), device_ms=round(ms, 3), kernel_ms=kernels, host_load_s=round(host_load, 2),
               mAP=float(res['ap'][0][-1, 0]), MOTA=float(res['metrics'][-4, 0]))
    if args.oracle:
        # the CPU baseline is the test oracle (numpy + scipy, single-threaded), timed on the same loaded frames
        O = importlib.import_module('oracle.poseval')
        t0 = time.time()
        (apAll, _, _), metrics, _ = O.evaluate_frames(copy.deepcopy(gt), copy.deepcopy(pr))
        out['oracle_s'] = round(time.time() - t0, 2)
        out['oracle_mAP'], out['oracle_MOTA'] = float(apAll[-1, 0]), float(metrics[-4, 0])
        assert abs(out['oracle_mAP'] - out['mAP']) <= 1e-12 * abs(out['mAP'])
        assert abs(out['oracle_MOTA'] - out['MOTA']) <= 1e-12 * abs(out['MOTA'])
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
