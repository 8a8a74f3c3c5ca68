"""Horizontally flipped training entries (lib/datasets/roidb.py:65-89 extend_with_flipped_entries,
lib/utils/keypoints.py:65-78 flip_keypoints, the flip map of lib/datasets/json_dataset.py:321-356 _init_keypoints)."""
import os

import numpy as np

from .boxes import flip_boxes

# keypoint index pairs swapped by a flip, in the order of the reference's keypoint lists: COCO's 17 joints
# (nose, left/right eye, ear, shoulder, elbow, wrist, hip, knee, ankle) and PoseTrack's (nose, head_bottom, head_top,
# left/right ear, shoulder, ...) share the indices.  Only datasets named keypoints_coco* swap the eyes and ears; every
# other dataset, PoseTrack included, keeps them (json_dataset.py:339-356, kept as the reference has it).
COCO_FLIP_PAIRS = ((1, 2), (3, 4), (5, 6), (7, 8), (9, 10), (11, 12), (13, 14), (15, 16))
DEFAULT_FLIP_PAIRS = ((5, 6), (7, 8), (9, 10), (11, 12), (13, 14), (15, 16))


def keypoint_flip_pairs(dataset_name):
    """The flip map _init_keypoints picks for a dataset name (a JSON roidb is named by its file's base name)."""
    return COCO_FLIP_PAIRS if os.path.basename(str(dataset_name)).startswith('keypoints_coco') else DEFAULT_FLIP_PAIRS


def flip_keypoints(gt_keypoints, flip_pairs, width, num_keypoints=None):
    """gt_keypoints [G, 3, K*T] (T frames of K joints) -> left / right joints swapped, x' = width - x - 1, and x = 0 where
    the visibility is 0 (the COCO convention)."""
    kps = np.asarray(gt_keypoints)
    K = num_keypoints or kps.shape[2]
    src = kps.reshape(kps.shape[0], 3, -1, K)
    out = src.copy()
    for l, r in flip_pairs:
        out[..., l] = src[..., r]
        out[..., r] = src[..., l]
    out = out.reshape(kps.shape)
    out[:, 0, :] = width - out[:, 0, :] - 1
    g, k = np.where(out[:, 2, :] == 0)
    out[g, 0, k] = 0
    return out


def flipped_entry(entry, flip_pairs, num_keypoints=None):
    """The mirrored copy of one roidb entry: boxes and keypoints flipped within the entry's original width, the other
    fields shared (segmentation masks are not carried)."""
    new = {k: v for k, v in entry.items() if k not in ('boxes', 'segms', 'gt_keypoints', 'flipped')}
    if 'boxes' in entry:
        new['boxes'] = flip_boxes(entry['boxes'], entry['width'])
    if 'gt_keypoints' in entry:
        new['gt_keypoints'] = flip_keypoints(entry['gt_keypoints'], flip_pairs, entry['width'], num_keypoints)
    new['flipped'] = True
    return new


def extend_with_flipped_entries(roidb, flip_pairs, num_keypoints=None):
    """roidb.py:65-89: append a flipped copy of every entry, after all the originals (in place, like the reference)."""
    roidb.extend([flipped_entry(e, flip_pairs, num_keypoints) for e in list(roidb)])
    return roidb


def training_roidb(dataset, flip):
    """The TRAIN.AUGMENT roidb of a dataset from core.test_engine.get_dataset (roidb.py:26-58 combined_roidb_for_training).
    flip (TRAIN.USE_FLIPPED): a flipped copy of every entry is appended after all the originals and BEFORE clip assembly,
    so utils/video.get_clip keys the clips by (video, frame, flipped).  A JSON list's per-frame entries are assembled into
    clips as dataset.get_roidb does; a synthetic entry carries no ground truth (tools/train_net.py draws it from the entry's
    seed), so its flipped copy only marks the entry flipped and keeps the seed: the same frames, mirrored on the device."""
    from ..core.config import cfg
    entries = getattr(dataset, 'entries', None)
    if not flip or entries is None:
        roidb = dataset.get_roidb(gt=True)
        return extend_with_flipped_entries(list(roidb), keypoint_flip_pairs(dataset.name)) if flip else roidb
    roidb = []
    for e in entries:
        e = dict(e)
        for k in ('boxes', 'gt_keypoints', 'tracks', 'gt_classes', 'is_crowd'):
            if k in e and not isinstance(e[k], np.ndarray):
                e[k] = np.asarray(e[k], dtype={'boxes': np.float32, 'is_crowd': bool}.get(k, np.int32))
        roidb.append(e)
    per_frame = cfg.MODEL.VIDEO_ON and roidb and not isinstance(roidb[0]['image'], (list, tuple))
    # a per-frame entry holds K joints; an entry that already carries its T frames holds K * T (NUM_KEYPOINTS per frame)
    extend_with_flipped_entries(roidb, keypoint_flip_pairs(dataset.name), None if per_frame else cfg.KRCNN.NUM_KEYPOINTS)
    if per_frame:
        from . import video
        roidb = video.get_clip(roidb)
    return roidb
