#!/usr/bin/env python
"""PoseTrack evaluation with the command line of the reference's poseval (lib/datasets/posetrack/poseval/py/evaluate.py):

    python tools/eval_posetrack.py -g GT_DIR -p PRED_DIR [-e] [-t] [-u]

-e prints the per-frame multi-person pose estimation AP table, -t the MOT table (MOTA per joint group, MOTP, precision,
recall), both as the reference's LaTeX rows; -u computes the MOT table's upper bound: every prediction a GT person selects
takes that person's GT track id, the others leave the MOT inputs (AP is unchanged).  Prediction files are the GT files' names in PRED_DIR.  The frame
assignment, AP and CLEAR-MOT accumulation run on the GPU (csrc/poseval.cu)."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def parse_args(argv=None):
    p = argparse.ArgumentParser(description='Evaluation of Pose Estimation and Tracking (PoseTrack)')
    p.add_argument('-g', '--groundTruth', required=False, type=str,
                   help='Directory containing ground truth annotatations per sequence in json format')
    p.add_argument('-p', '--predictions', required=False, type=str,
                   help='Directory containing predictions per sequence in json format')
    p.add_argument('-e', '--evalPoseEstimation', required=False, action='store_true',
                   help='Evaluation of per-frame  multi-person pose estimation using AP metric')
    p.add_argument('-t', '--evalPoseTracking', required=False, action='store_true',
                   help='Evaluation of video-based  multi-person pose tracking using MOT metrics')
    p.add_argument('-u', '--trackUpperBound', required=False, action='store_true',
                   help='Compute an upper bound on the tracking by using GT track ids.')
    return p.parse_args(argv)


def main(argv=None):
    from detectandtrack_b200.datasets import posetrack_eval as E
    args = parse_args(argv)
    if not args.groundTruth or not args.predictions:
        raise SystemExit('both -g GT_DIR and -p PRED_DIR are needed')
    print(args)
    print('Loading data')
    gtFramesAll, prFramesAll, names = E.load_data_dir(args.groundTruth, args.predictions)
    print('# gt frames  :', len(gtFramesAll))
    print('# pred frames:', len(prFramesAll))
    res = E.evaluate_pack(E.PoseTrackPack(gtFramesAll, prFramesAll, names), args.evalPoseEstimation, args.evalPoseTracking,
                          track_upper_bound=args.trackUpperBound)
    if args.evalPoseEstimation:
        print('Evaluation of per-frame multi-person pose estimation')
        print('Average Precision (AP) metric:')
        E.print_table(res['ap'][0])
    if args.evalPoseTracking:
        print('Evaluation of video-based  multi-person pose tracking')
        print('Multiple Object Tracking (MOT) metrics:')
        E.print_table(res['metrics'], motHeader=True)
    return res


if __name__ == '__main__':
    main()
