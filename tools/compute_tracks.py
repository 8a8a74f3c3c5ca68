#!/usr/bin/env python
"""Tracking entry point with the reference's command line (tools/compute_tracks.py:26-52):

    python tools/compute_tracks.py --cfg X.yaml [KEY VALUE ...]
Loads <output_dir>/detections.pkl (or TRACKING.DETECTIONS_FILE), links detections per video
on the GPU and writes detections_withTracks.pkl and the PoseTrack JSON of every video; with
EVAL.POSETRACK_ANNOTATION_DIR set, scores them (total mAP and MOTA) on the GPU."""
import argparse
import logging
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from detectandtrack_b200.core.config import cfg, cfg_from_file, cfg_from_list, assert_and_infer_cfg, get_output_dir  # noqa: E402


def parse_args():
    p = argparse.ArgumentParser()
    p.add_argument('--cfg', dest='cfg_file', required=True, help='Config file')
    p.add_argument('opts', help='See core/config.py for all options', default=None, nargs=argparse.REMAINDER)
    return p.parse_args()


def main():
    from detectandtrack_b200.core.test_engine import get_roidb_and_dataset
    from detectandtrack_b200.core.tracking_engine import run_posetrack_tracking
    args = parse_args()
    cfg_from_file(args.cfg_file)
    if args.opts:
        cfg_from_list(args.opts)
    assert_and_infer_cfg()
    test_output_dir = get_output_dir(training=False)
    json_data, dataset, _, _, _ = get_roidb_and_dataset(None, include_gt=True)
    run_posetrack_tracking(test_output_dir, json_data, dataset=dataset)


if __name__ == '__main__':
    logging.basicConfig(level=logging.INFO, format='%(levelname)s %(filename)s:%(lineno)4d: %(message)s', stream=sys.stdout)
    main()
