"""Golden vectors for the TRAIN.AUGMENT minibatch (flipped roidb entries, per-clip training scale), from the REFERENCE's own
modules.  Build container only (needs /root/reference):

    python tests/golden/gen_golden_train_aug.py      -> tests/golden/train_aug.npz

What runs, unmodified, from /root/reference/lib:
    datasets/roidb.py          extend_with_flipped_entries (+ utils/keypoints.py flip_keypoints, utils/segms.py flip_segms)
    datasets/json_dataset.py   JsonDataset._init_keypoints, on a stub dataset whose COCO categories list the PoseTrack
                               or the COCO keypoint names (it picks the flip map from the dataset name)
    utils/boxes.py             flip_boxes (it asserts 4 columns, so a T-frame tube is flipped frame by frame)
    utils/video.py             get_clip over the flipped-extended per-frame roidb
    roi_data/minibatch.py      _get_image_blob (+ utils/blob.py prep_im_for_blob, im_list_to_blob)
Shims, all recorded here: those of gen_golden_video (gen_golden._setup_reference_imports, stub cPickle / h5py / caffe2.*
modules, tqdm -> identity); utils/image.read_image_video returns seeded frames instead of reading files; prep_im_for_blob
is wrapped to record each clip's resized shape (its result is passed through).  The ONE behavioural patch:
`numpy.random.randint` is the counter-based draw of oracle/targets.py on stream 5 (the training scale), so scale index j of
the minibatch is randint(len(SCALES)) at counter j — what tools/train_net.py draws at iteration 0 on rank 0.
"""
import os
import pickle
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

SEED = 7
POSETRACK_KEYPOINTS = ['nose', 'head_bottom', 'head_top', 'left_ear', 'right_ear', 'left_shoulder', 'right_shoulder',
                       'left_elbow', 'right_elbow', 'left_wrist', 'right_wrist', 'left_hip', 'right_hip', 'left_knee',
                       'right_knee', 'left_ankle', 'right_ankle']
COCO_KEYPOINTS = ['nose', 'left_eye', 'right_eye', 'left_ear', 'right_ear', 'left_shoulder', 'right_shoulder', 'left_elbow',
                  'right_elbow', 'left_wrist', 'right_wrist', 'left_hip', 'right_hip', 'left_knee', 'right_knee', 'left_ankle',
                  'right_ankle']
# _get_image_blob case: two clips of T = 2 frames at two source sizes (landscape, portrait), the first one flipped
BLOB_SIZES = ((60, 80), (90, 50))
BLOB_FLIPPED = (True, False)
BLOB_SCALES = (48, 64, 72)
BLOB_MAX_SIZE = 100
BLOB_T = 2


def frame_roidb(seed=5):
    """A per-frame PoseTrack-like roidb: two videos, a missing frame, joints with visibility 0."""
    rng = np.random.RandomState(seed)
    roidb = []
    for v, nf, (H, W) in (('vidA', 4, (240, 320)), ('vidB', 3, (300, 200))):
        for f in range(1, nf + 1):
            if v == 'vidA' and f == 3:
                continue
            ids = sorted(rng.choice(5, size=rng.randint(1, 4), replace=False).tolist())
            n = len(ids)
            x1 = rng.uniform(0, W - 40, n); y1 = rng.uniform(0, H - 40, n)
            boxes = np.stack([x1, y1, x1 + rng.uniform(5, 38, n), y1 + rng.uniform(5, 38, n)], 1).astype(np.float32)
            kps = rng.randint(0, min(H, W), (n, 3, 17)).astype(np.int32)
            kps[:, 2] = rng.randint(0, 3, (n, 17))
            kps[0, 2, :4] = 0                                          # invisible joints: x goes to 0 after the flip
            roidb.append(dict(image='%s/%06d.jpg' % (v, f), frame_id=f, flipped=False, height=H, width=W, id=len(roidb), nframes=nf,
                              is_labeled=True, has_visible_keypoints=True, tracks=np.array(ids, np.int32).reshape(-1, 1),
                              boxes=boxes, gt_keypoints=kps, gt_classes=np.ones(n, np.int32), is_crowd=np.zeros(n, bool),
                              segms=[[] for _ in range(n)], box_to_gt_ind_map=np.arange(n, dtype=np.int32),
                              max_classes=np.ones(n, np.int64), max_overlaps=np.ones(n, np.float32), seg_areas=np.ones(n, np.float32),
                              head_boxes=-np.ones((n, 4), np.float32)))
    return roidb


def tube_boxes(seed=6, n=5, T=3, width=320):
    rng = np.random.RandomState(seed)
    x1 = rng.uniform(0, width - 50, (n, T)); y1 = rng.uniform(0, 200, (n, T))
    b = np.stack([x1, y1, x1 + rng.uniform(1, 49, (n, T)), y1 + rng.uniform(1, 40, (n, T))], 2)
    return b.reshape(n, 4 * T).astype(np.float32), width


def blob_frames(seed=8):
    rng = np.random.RandomState(seed)
    return [rng.randint(0, 256, (BLOB_T, h, w, 3)).astype(np.uint8) for h, w in BLOB_SIZES]


def main():
    import gen_golden as g
    import gen_golden_targets as gt
    g._setup_reference_imports()
    sys.modules['cPickle'] = pickle
    for n in ['caffe2.proto.caffe2_pb2', 'caffe2.python.scope', 'caffe2.python.core', 'caffe2.python.workspace',
              'caffe2.python.utils', 'h5py', 'pycocotools.mask', 'pycocotools.coco']:
        gt._stub(n)
    sys.modules['pycocotools.coco'].COCO = object
    import scipy.sparse
    import tqdm
    tqdm.tqdm = lambda x, **kw: x
    from oracle import targets as ot
    import numpy.random as npr
    from core.config import cfg
    import utils.video as rv
    rv.tqdm = lambda x, **kw: x
    import utils.boxes as rbox
    import datasets.json_dataset as jd
    import datasets.roidb as rroidb
    out = {}

    # ------------------------------------------------------------------ flipped entries, both flip maps
    class _Cats(object):
        def __init__(self, names):
            self.names = names

        def loadCats(self, ids):
            return [{'name': 'person', 'keypoints': list(self.names)}]

    class _DS(object):
        frames_from_video = False

    for tag, name, names in (('posetrack', 'posetrack_v1.0_train', POSETRACK_KEYPOINTS), ('coco', 'keypoints_coco_2014_train', COCO_KEYPOINTS)):
        ds = _DS()
        ds.category_to_id_map = {'person': 1}
        ds.COCO = _Cats(names)
        jd.JsonDataset._init_keypoints(ds, name=name)
        roidb = frame_roidb()
        n0 = len(roidb)
        rroidb.extend_with_flipped_entries(roidb, ds)
        out[tag + '_n'] = np.int32(len(roidb))
        pairs = sorted((names.index(l), names.index(r)) for l, r in ds.keypoint_flip_map.items())
        out[tag + '_pairs'] = np.array(pairs, np.int32)
        for i, e in enumerate(roidb[n0:]):
            out['%s_%d_boxes' % (tag, i)] = e['boxes']
            out['%s_%d_kps' % (tag, i)] = e['gt_keypoints']
            assert e['flipped'] is True and e['width'] == roidb[i]['width']
        if tag == 'posetrack':
            # clip assembly over the extended roidb: flipped frames only join flipped clips
            cfg.VIDEO.NUM_FRAMES, cfg.VIDEO.NUM_FRAMES_MID, cfg.VIDEO.TIME_INTERVAL = 3, 1, 1
            for e in roidb:
                e['dataset'] = _DS()
                e['gt_overlaps'] = scipy.sparse.csr_matrix(np.tile(np.array([[0., 1.]], np.float32), (len(e['boxes']), 1)))
            res = rv.get_clip(roidb, remove_imperfect=False)
            out['clip_n'] = np.int32(len(res))
            for i, e in enumerate(res):
                out['clip_%d_image' % i] = np.array(e['image'])
                out['clip_%d_flipped' % i] = np.bool_(e['flipped'])
                for k in ('tracks', 'boxes', 'gt_keypoints', 'track_visible'):
                    out['clip_%d_%s' % (i, k)] = e[k]

    # ------------------------------------------------------------------ flip_boxes on T = 3 tubes (frame by frame)
    tubes, width = tube_boxes()
    out['tubes_in'], out['tubes_width'] = tubes, np.int32(width)
    out['tubes_flipped'] = np.concatenate([rbox.flip_boxes(tubes[:, 4 * t:4 * t + 4], width) for t in range(3)], 1)

    # ------------------------------------------------------------------ _get_image_blob: per-clip scale draw + flip
    def p_randint(low, high=None, size=None, dtype=int):
        assert low == 0 and high is not None
        return ot.randint(high, size, SEED, 5, 0)
    npr.randint = p_randint
    import utils.blob as blob_utils
    import utils.image as image_utils
    import roi_data.minibatch as mb
    frames = blob_frames()
    image_utils.read_image_video = lambda entry: [f for f in frames[entry['clip']]]
    shapes = []
    prep = blob_utils.prep_im_for_blob

    def rec_prep(im, means, targets, max_size):
        ims, scales = prep(im, means, targets, max_size)
        shapes.append(ims[0].shape[:2])
        return ims, scales
    blob_utils.prep_im_for_blob = rec_prep
    cfg.TRAIN.SCALES, cfg.TRAIN.MAX_SIZE = BLOB_SCALES, BLOB_MAX_SIZE
    cfg.FPN.FPN_ON, cfg.FPN.COARSEST_STRIDE = True, 32
    cfg.MODEL.VIDEO_ON, cfg.VIDEO.NUM_FRAMES = True, BLOB_T
    roidb = [dict(clip=b, flipped=BLOB_FLIPPED[b], height=h, width=w) for b, (h, w) in enumerate(BLOB_SIZES)]
    blob, im_scales = mb._get_image_blob(roidb)
    draws = ot.randint(len(BLOB_SCALES), len(roidb), SEED, 5, 0)
    out['blob'] = blob.astype(np.float32)                                 # [B, 3, T, Hp, Wp]
    out['blob_im_scales'] = np.array(im_scales, np.float64)
    out['blob_targets'] = np.array([BLOB_SCALES[d] for d in draws], np.int32)
    out['blob_resized'] = np.array(shapes[::BLOB_T], np.int32)           # one (hr, wr) per clip
    assert all(shapes[b * BLOB_T] == shapes[b * BLOB_T + t] for b in range(len(roidb)) for t in range(BLOB_T))
    out['blob_frames0'], out['blob_frames1'] = frames
    np.savez_compressed(os.path.join(HERE, 'train_aug.npz'), **out)
    print('wrote train_aug.npz', len(out), 'targets', out['blob_targets'], 'scales', im_scales, 'resized', out['blob_resized'])


if __name__ == '__main__':
    main()
