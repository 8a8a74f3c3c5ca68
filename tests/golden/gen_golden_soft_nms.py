"""Golden vectors for soft-NMS and bounding-box voting, from the REFERENCE's own functions.  Needs the reference
checkout that oracle/build_ref.py compiles from:

    python tests/golden/gen_golden_soft_nms.py      -> tests/golden/soft_nms.npz

What runs, unmodified, from the reference's lib/:
    utils/cython_nms.pyx  soft_nms, compiled by oracle/build_ref.py (oracle/_ref/cython_nms)
    utils/boxes.py        box_voting (with bbox_overlaps over the compiled cython_bbox)
Shims: those of gen_golden_tta (gen_golden._setup_reference_imports, stub caffe2.* / pycocotools modules).

Soft-NMS cases s<k>: dets, params (sigma, Nt, threshold, method) -> rows, inds.  Each input set runs all three methods
at two sigmas.  Vote cases v<k>: top, all, thresh -> voted.
"""
import os
import pickle
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
F32 = np.float32


def _realistic(rng, n, w=640, h=480):
    cx, cy = rng.uniform(0, w, 12), rng.uniform(0, h, 12)              # a few objects, many proposals each
    k = rng.randint(0, 12, n)
    bw, bh = rng.uniform(20, 160, 12)[k], rng.uniform(40, 240, 12)[k]
    x1 = cx[k] - bw / 2 + rng.normal(0, 6, n); y1 = cy[k] - bh / 2 + rng.normal(0, 6, n)
    x2 = x1 + bw * rng.uniform(0.8, 1.2, n); y2 = y1 + bh * rng.uniform(0.8, 1.2, n)
    x1, x2 = np.clip(x1, 0, w - 1), np.clip(x2, 0, w - 1)
    y1, y2 = np.clip(y1, 0, h - 1), np.clip(y2, 0, h - 1)
    s = rng.uniform(0.05, 1.0, n)
    return np.stack([x1, y1, x2, y2, s], 1).astype(F32)


def soft_inputs(seed=5):
    rng = np.random.RandomState(seed)
    sets = [_realistic(rng, 300), _realistic(rng, 120)]
    # exact-duplicate boxes and score ties (discards permute the survivors, which decides later ties)
    sets.append(np.array([[0, 0, 9, 9, .9], [0, 0, 9, 9, .9], [20, 20, 29, 29, .9], [0, 0, 9, 9, .9],
                          [1, 1, 10, 10, .9], [20, 20, 29, 29, .5], [0, 0, 9, 9, .5]], F32))
    dup = _realistic(rng, 40)
    dup[20:] = dup[:20]
    dup[::3, 4] = F32(0.5)
    sets.append(dup)
    # ov == Nt: with the '+1' convention [0 0 9 4] and [0 0 19 9] overlap [0 0 9 9] by exactly .5, [0 0 9 2] by fp32(.3)
    a = [0, 0, 9, 9]
    sets.append(np.array([a + [.9], [0, 0, 9, 4, .8], [0, 0, 9, 2, .7], [5, 0, 14, 9, .6], [0, 0, 19, 9, .5]], F32))
    # scores that decay to just under and exactly to 1e-4: score s, linear weight (1 - ov) with ov = .5 -> s / 2
    t = F32(0.0001)
    sets.append(np.array([a + [.9], [0, 0, 9, 4, 2 * t], [0, 0, 9, 4, np.nextafter(2 * t, F32(0))],
                          [0, 0, 9, 4, np.nextafter(2 * t, F32(1))], [0, 0, 9, 4, t], [40, 40, 49, 49, F32(5e-5)]], F32))
    # degenerate boxes (iw <= 0 / ih <= 0, negative widths) and negative coordinates
    deg = _realistic(rng, 60)
    deg[:10, 2] = deg[:10, 0] - 3
    deg[10:20, 3] = deg[10:20, 1] - 1
    deg[20:40, :4] -= F32(700)
    sets.append(deg)
    sets.append(np.zeros((0, 5), F32))
    sets.append(_realistic(rng, 1))
    return sets


SOFT_PARAMS = [(sig, nt, th, m) for m in (0, 1, 2) for sig, nt, th in ((0.5, 0.3, 0.0001), (0.1, 0.5, 0.001))]


def vote_inputs(seed=7):
    rng = np.random.RandomState(seed)
    out = []
    for n_match in (1, 9, 129, 1100):
        alld = _realistic(rng, 40)
        alld[:, :4] += F32(1000)                                       # nothing near the cluster
        base = np.array([100, 120, 180, 260], F32)
        cl = base + rng.normal(0, 1.5, (n_match, 4)).astype(F32)
        cl = np.concatenate([cl, rng.uniform(0.05, 1, (n_match, 1))], 1).astype(F32)
        alld = np.concatenate([alld[:20], cl, alld[20:]]).astype(F32)
        top = np.concatenate([np.append(base, F32(0.99))[None], alld[:3], alld[25:27]]).astype(F32)
        out.append((top, alld, 0.8))
    alld = _realistic(rng, 500)
    out.append((alld[:60], alld, 0.8))
    out.append((alld[:60], alld, 0.5))
    return out


def main():
    import gen_golden as g
    import gen_golden_targets as gt
    g._setup_reference_imports()
    sys.modules['cPickle'] = pickle
    for n in ['caffe2.proto.caffe2_pb2', 'caffe2.python.scope', 'caffe2.python.core', 'caffe2.python.workspace',
              'caffe2.python.utils', 'h5py', 'pycocotools.mask', 'pycocotools.coco']:
        gt._stub(n)
    from oracle._ref import cython_nms
    import utils.boxes as rbox
    out = {}
    k = 0
    for d in soft_inputs():
        for sig, nt, th, m in SOFT_PARAMS:
            rows, inds = cython_nms.soft_nms(np.ascontiguousarray(d), F32(sig), F32(nt), F32(th), np.uint8(m))
            out['s%d_dets' % k] = d
            out['s%d_params' % k] = np.array([sig, nt, th, m], F32)
            out['s%d_rows' % k] = np.asarray(rows, F32).reshape(-1, 5)
            out['s%d_inds' % k] = np.asarray(inds, np.int64)
            k += 1
    for j, (top, alld, th) in enumerate(vote_inputs()):
        out['v%d_top' % j], out['v%d_all' % j], out['v%d_thresh' % j] = top, alld, F32(th)
        out['v%d_voted' % j] = rbox.box_voting(top, alld, th).astype(F32)
    np.savez_compressed(os.path.join(HERE, 'soft_nms.npz'), **out)
    print('wrote soft_nms.npz: %d soft-NMS cases, %d vote cases, %d bytes'
          % (k, j + 1, os.path.getsize(os.path.join(HERE, 'soft_nms.npz'))))


if __name__ == '__main__':
    main()
