"""Golden vectors for test-time augmentation's flip and combine, from the REFERENCE's own functions.  Build container only
(needs /root/reference):

    python tests/golden/gen_golden_tta.py      -> tests/golden/tta.npz

What runs, unmodified, from /root/reference/lib:
    utils/boxes.py       flip_boxes, on every 4-column class slice of seeded box-head rows [R, 4C] (it asserts 4 columns)
    utils/keypoints.py   flip_heatmaps (the COCO joint swap of get_keypoints, then the x mirror)
    lib/core/test.py     the combine of im_detect_keypoints_aug (:737-744) restated as its two numpy calls, np.mean and
                         np.amax over axis 0 of the per-view maps (that function also runs the network)
Shims: those of gen_golden (gen_golden._setup_reference_imports, stub cPickle / caffe2.* / pycocotools modules).
"""
import os
import pickle
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

BOX_ROWS, BOX_CLASSES, WIDTH = 64, 3, 320
HM_ROIS, HM_K, HM_M, HM_VIEWS = 2, 17, 8, 3          # the flip and combine do not depend on the map size


def inputs(seed=11):
    rng = np.random.RandomState(seed)
    x1 = rng.uniform(0, WIDTH - 1, (BOX_ROWS, BOX_CLASSES)); y1 = rng.uniform(0, 200, (BOX_ROWS, BOX_CLASSES))
    x2 = np.minimum(x1 + rng.uniform(0, 80, x1.shape), WIDTH - 1); y2 = y1 + rng.uniform(0, 60, y1.shape)
    boxes = np.stack([x1, y1, x2, y2], 2).reshape(BOX_ROWS, 4 * BOX_CLASSES).astype(np.float32)
    maps = rng.standard_normal((HM_VIEWS, HM_ROIS, HM_K, HM_M, HM_M)).astype(np.float32) * 3
    maps[1, 0, 0, :4, :4] = maps[0, 0, 0, :4, :4]                 # exact ties between views
    return boxes, maps


def main():
    import gen_golden as g
    import gen_golden_targets as gt
    g._setup_reference_imports()
    sys.modules['cPickle'] = pickle
    for n in ['caffe2.proto.caffe2_pb2', 'caffe2.python.scope', 'caffe2.python.core', 'caffe2.python.workspace',
              'caffe2.python.utils', 'h5py', 'pycocotools.mask', 'pycocotools.coco']:
        gt._stub(n)
    import utils.boxes as rbox
    import utils.keypoints as rkp
    boxes, maps = inputs()
    out = dict(boxes=boxes, width=np.int32(WIDTH), maps=maps)
    out['boxes_flipped'] = np.concatenate([rbox.flip_boxes(boxes[:, 4 * j:4 * j + 4], WIDTH) for j in range(BOX_CLASSES)], 1)
    views = [maps[0], rkp.flip_heatmaps(maps[1]), maps[2]]        # views 1 flipped
    out['maps_flip1'] = np.ascontiguousarray(views[1])
    out['hm_avg'] = np.mean(views, axis=0)
    out['hm_max'] = np.amax(views, axis=0)
    np.savez_compressed(os.path.join(HERE, 'tta.npz'), **out)
    print('wrote tta.npz', {k: v.shape for k, v in out.items()})


if __name__ == '__main__':
    main()
