"""PoseTrack result writer — the step right after tracking (SURVEY.md §8(f) rank 2), mirroring the surface of
the reference's ``core.mpii_eval_engine`` (lib/core/mpii_eval_engine.py):

    coco2posetrack(preds, src_kps, dst_kps, global_score, kp_conf_type)      :103-150
    _convert_data_to_annorect_struct(boxes, poses, tracks)                    :153-183
    _run_posetrack_eval(roidb, det_file, dataset, output_dir)                 :246-314  (JSON writing part)
    run_mpii_eval(test_output_dir, roidb, dataset)                            :317-337

    video2filenames(pathtodir)                                                :184-205
    _run_eval(annot_dir, output_dir, eval_tracking, eval_pose)               :208-216

What it does: per detection, remap the 17 COCO-order keypoints (x, y, logit) of ``detections_withTracks.pkl``
to the 15 PoseTrack/MPII joints (neck = mid-shoulder, head_top = nose reflected about the neck), attach the
track id and write one ``{'annolist': [...]}`` JSON per video.  ``run_mpii_eval`` then scores the files: with an
``evaluator`` handed in, by calling it; else, when the dataset has an ``annotation_directory`` (a dataset without
one takes EVAL.POSETRACK_ANNOTATION_DIR), with the device PoseTrack evaluation (datasets/posetrack_eval.py), logging
(total mAP, total MOTA) and, with EVAL.EVAL_MPII_PER_VIDEO, writing ``<det_file>_per_video_scores.txt``.

Arithmetic note: the reference runs on numpy 1.14, where ``float32_scalar / 2.0`` and ``float32_scalar *
python_float`` promote to float64.  The sums of two float32 values are therefore rounded in fp32 and everything
after that is done in double, which is what this file does explicitly (numpy >= 2 would keep fp32).
"""
import json
import logging
import os
import os.path as osp
import pickle
import time

import numpy as np

from .config import cfg

logger = logging.getLogger(__name__)

# joint orders (mpii_eval_engine.py:36-92): the detector's order, PoseTrack's 17-name order and the 15 MPII
# joints the PoseTrack evaluation expects
coco_src_keypoints = [
    'nose', 'left_eye', 'right_eye', 'left_ear', 'right_ear', 'left_shoulder', 'right_shoulder', 'left_elbow',
    'right_elbow', 'left_wrist', 'right_wrist', 'left_hip', 'right_hip', 'left_knee', 'right_knee', 'left_ankle',
    'right_ankle']
posetrack_src_keypoints = [
    'nose', 'head_bottom', 'head_top', 'left_ear', 'right_ear', 'left_shoulder', 'right_shoulder', 'left_elbow',
    'right_elbow', 'left_wrist', 'right_wrist', 'left_hip', 'right_hip', 'left_knee', 'right_knee', 'left_ankle',
    'right_ankle']
dst_keypoints = [
    'right_ankle', 'right_knee', 'right_hip', 'left_hip', 'left_knee', 'left_ankle', 'right_wrist', 'right_elbow',
    'right_shoulder', 'left_shoulder', 'left_elbow', 'left_wrist', 'neck', 'nose', 'head_top']


def _compute_score(conf, global_conf, kp_conf_type=None):
    """:87-100.  'global': the detection score, 'local': the keypoint logit, 'scaled': their product."""
    kp_conf_type = cfg.TRACKING.KP_CONF_TYPE if kp_conf_type is None else kp_conf_type
    if kp_conf_type == 'global':
        return global_conf
    if kp_conf_type == 'local':
        return conf
    if kp_conf_type == 'scaled':
        return conf * global_conf
    raise NotImplementedError('Uknown type {}'.format(kp_conf_type))


def _half_sum(a, b):
    """(a + b) / 2.0 as the reference evaluates it: fp32 sum, then a double division."""
    return float(np.float32(a) + np.float32(b)) / 2.0


def coco2posetrack(preds, src_kps, dst_kps, global_score, kp_conf_type=None):
    """preds [>=3, K] rows (x, y, logit, ...) in ``src_kps`` order -> list of PoseTrack point dicts in
    ``dst_kps`` order.  Joints whose local score is below EVAL.EVAL_MPII_KPT_THRESHOLD are dropped."""
    preds = np.asarray(preds)
    where = {name: i for i, name in enumerate(src_kps)}
    thr = cfg.EVAL.EVAL_MPII_KPT_THRESHOLD
    global_score = float(global_score)
    points = []
    for k, name in enumerate(dst_kps):
        if name in where:
            i = where[name]
            x, y = float(preds[0, i]), float(preds[1, i])
            local = _half_sum(preds[2, i], preds[2, i])
        elif name in ('neck', 'head_top'):
            r, l = where['right_shoulder'], where['left_shoulder']
            x, y = _half_sum(preds[0, r], preds[0, l]), _half_sum(preds[1, r], preds[1, l])
            local = _half_sum(preds[2, r], preds[2, l])
            if name == 'head_top':                      # the nose reflected about the mid-shoulder point
                n = where['nose']
                xn, yn = float(preds[0, n]), float(preds[1, n])
                x, y = xn - (x - xn), yn - (y - yn)
        else:
            continue
        if local >= thr:
            points.append({'id': [k], 'x': [x], 'y': [y], 'score': [_compute_score(local, global_score, kp_conf_type)]})
    return points


def _convert_data_to_annorect_struct(boxes, poses, tracks):
    """boxes [N, 5] (score last), poses: N arrays [4, 17], tracks: N ids -> the frame's 'annorect' list.
    Detections under EVAL.EVAL_MPII_DROP_DETECTION_THRESHOLD are dropped; an empty frame gets the dummy
    prediction the MOTA code needs (:170-182)."""
    boxes = np.asarray(boxes)
    annorect = []
    for j in range(boxes.shape[0]):
        score = boxes[j, -1]
        if score < cfg.EVAL.EVAL_MPII_DROP_DETECTION_THRESHOLD:
            continue
        annorect.append({'annopoints': [{'point': coco2posetrack(poses[j], posetrack_src_keypoints, dst_keypoints, score)}],
                         'score': [float(score)], 'track_id': [tracks[j]]})
    if boxes.shape[0] == 0:
        annorect.append({'annopoints': [{'point': [{'id': [0], 'x': [0], 'y': [0], 'score': [-100.0]}]}],
                         'score': [0], 'track_id': [0]})
    return annorect


def _image_path(entry):
    im = entry['image']
    return im[len(im) // 2] if isinstance(im, (list, tuple)) else im      # utils/image.py:44-48


def _frame_number(image_name, entry):
    """PoseTrack frames are named by their number (:262); other datasets fall back to the roidb's frame id."""
    try:
        return int(osp.basename(image_name).split('.')[0])
    except ValueError:
        return int(entry.get('frame_id', 0))


def build_annolists(roidb, dets, image_directory=''):
    """Group the per-image results by video (dirname of the image path below ``image_directory``):
    {video_name: [ {'image', 'imagenum', 'annorect'}, ... ]} in roidb order (:256-281)."""
    assert len(roidb) == len(dets['all_boxes'][1]), 'Mismatch {} vs {}'.format(len(roidb), len(dets['all_boxes'][1]))
    has_tracks = 'all_tracks' in dets
    out = {}
    for i, entry in enumerate(roidb):
        image_name = _image_path(entry)[len(image_directory):]
        kps = dets['all_keyps'][1][i]
        tracks = dets['all_tracks'][1][i] if has_tracks else [1] * len(kps)
        out.setdefault(osp.dirname(image_name), []).append({
            'image': image_name,
            'imagenum': [_frame_number(image_name, entry)],
            'annorect': _convert_data_to_annorect_struct(dets['all_boxes'][1][i], kps, tracks)})
    return out


def write_posetrack_json(roidb, dets, output_dir, image_directory='', out_filenames=None):
    """One JSON per video.  ``out_filenames`` maps 'images/<video>' to the annotation file name (the reference
    derives it from the dataset's annotation directory, :185-207); without it the file is '<video>.json' with
    path separators replaced."""
    os.makedirs(output_dir, exist_ok=True)
    for f in os.listdir(output_dir):                       # previous predictions, if any (:284)
        if f.endswith('.json'):
            os.remove(osp.join(output_dir, f))
    paths = {}
    for vname, vdata in build_annolists(roidb, dets, image_directory).items():
        key = osp.join('images', vname)
        fname = out_filenames[key] if out_filenames is not None else (vname.strip('/').replace('/', '_') or 'video') + '.json'
        paths[vname] = osp.join(output_dir, fname)
        with open(paths[vname], 'w') as fout:
            json.dump({'annolist': vdata}, fout)
    logger.info('Wrote all predictions in JSON to %s', output_dir)
    return paths


def video2filenames(pathtodir):
    """:184-205.  {video directory: output JSON name} from the PoseTrack .mat annotations of ``pathtodir``."""
    import scipy.io as sio
    output = {}
    for fname in os.listdir(pathtodir):
        if not (osp.isfile(osp.join(pathtodir, fname)) and '.mat' in fname):
            continue
        data = sio.loadmat(osp.join(pathtodir, fname), squeeze_me=True, struct_as_record=False)
        output[osp.dirname(data['annolist'][0].image.name)] = fname.replace('.mat', '.json')
    return output


def _run_eval(annot_dir, output_dir, eval_tracking=False, eval_pose=True, per_video=False):
    """:208-216.  (total mAP, total MOTA) of the JSON files of ``output_dir`` against ``annot_dir``; with per_video
    also {file name: (mAP, MOTA)} as each file scores on its own (NaN for both where that fails)."""
    from ..datasets import posetrack_eval
    run = posetrack_eval.evaluate_upper_bound if cfg.TRACKING.DEBUG.UPPER_BOUND_4_EVAL_UPPER_BOUND else posetrack_eval.evaluate
    res = run(annot_dir, output_dir, eval_pose, eval_tracking, per_video=per_video)
    (apAll, _, _), mota = res[0], res[1]
    return (apAll[-1][0], mota[-4][0]) + tuple(res[2:])


def _write_per_video_scores(path, paths, videos):
    """:292-314: one 'video ap mota' line per video, sorted on the AP with Python's sorted."""
    res = [(vname,) + tuple(videos.get(osp.basename(p), (np.nan, np.nan))) for vname, p in paths.items()]
    res = sorted(res, key=lambda x: x[1])
    logger.info('Writing per-video scores to %s', path)
    with open(path, 'w') as fout:
        for el in res:
            fout.write('{} {} {}\n'.format(el[0], el[1], el[2]))


def _run_posetrack_eval(roidb, det_file, dataset, output_dir, evaluator=None):
    with open(det_file, 'rb') as fin:
        try:
            dets = pickle.load(fin)
        except UnicodeDecodeError:                       # pickles written by the py2 reference
            fin.seek(0)
            dets = pickle.load(fin, encoding='latin1')
    # a dataset without its own directories takes EVAL.POSETRACK_IMAGE_DIR / EVAL.POSETRACK_ANNOTATION_DIR ('' by default)
    image_directory = getattr(dataset, 'image_directory', cfg.EVAL.POSETRACK_IMAGE_DIR) if dataset is not None else ''
    out_filenames = getattr(dataset, 'out_filenames', None) if dataset is not None else None
    annot_dir = getattr(dataset, 'annotation_directory', cfg.EVAL.POSETRACK_ANNOTATION_DIR) if dataset is not None else ''
    if evaluator is None and annot_dir and out_filenames is None and \
            any(f.endswith('.mat') for f in os.listdir(annot_dir)):
        out_filenames = video2filenames(annot_dir)
    paths = write_posetrack_json(roidb, dets, output_dir, image_directory, out_filenames)
    if evaluator is not None:
        return paths, evaluator(getattr(dataset, 'annotation_directory', None), output_dir, 'all_tracks' in dets)
    if not annot_dir:
        logger.info('No evaluator given and no annotation directory (EVAL.POSETRACK_ANNOTATION_DIR): '
                    'the PoseTrack JSON files are written, not scored')
        return paths, None
    eval_tracking = 'all_tracks' in dets
    logger.info('Running dataset level evaluation...')
    st_time = time.time()
    res = _run_eval(annot_dir, output_dir, eval_tracking, per_video=cfg.EVAL.EVAL_MPII_PER_VIDEO)
    logger.info('(total mAP, total MOTA) = %r', (float(res[0]), float(res[1])))
    logger.info('...Done in %s', time.time() - st_time)
    if cfg.EVAL.EVAL_MPII_PER_VIDEO:                     # every video scored alone, in the same device launches
        _write_per_video_scores(osp.join(osp.dirname(osp.normpath(output_dir)), osp.basename(det_file) + '_per_video_scores.txt'),
                                paths, res[2])
    return paths, res[:2]


def run_mpii_eval(test_output_dir, roidb, dataset=None, evaluator=None):
    """:317-337.  Looks for detections_withTracks.pkl, writes '<file>_json/' next to it."""
    det_file = osp.join(test_output_dir, 'detections_withTracks.pkl')
    if not osp.exists(det_file):
        logger.warning('No detection files found from %s', [det_file])
        return None
    logger.info('Evaluating %s', det_file)
    return _run_posetrack_eval(roidb, det_file, dataset, osp.join(test_output_dir, osp.basename(det_file) + '_json/'),
                               evaluator)
