"""GPU: every launch key of the dense ops on the benchmarked steps (dt_roi_align, dt_roi_align_bwd, dt_maxpool2d, dt_prep_clip,
dt_keypoint_decode, dt_spatial_mean, dt_fold_tube_heads, dt_scale_rois), launched at the step's shapes on random data and
compared with the fp64 references of tests/test_dense_reference.py, plus a coverage test that proves the table lists every key
that DetectionEngine.detect (r50fpn3d, r50fpn2d, r18tube, every dtype the engine takes) and KeypointRcnnTrainer.step launch.

Tolerances are derived next to each assert (u = 2^-24).  Nothing is tuned to pass."""
import numpy as np
import pytest
import torch

from test_dense_reference import (F32, U24, RoiAlignMatrix, cubic_matrix, fold_tube_heads_ref, join, keypoint_maps_ref,
                                  keypoints_from_maps, linear_abs, maxpool_ref, pairs, prep_ref, round_tf32, scale_rois_ref,
                                  spatial_mean_seq, split_bf16, upsample2x_matrix)

pytestmark = pytest.mark.gpu

K_COORD = 4     # ulps a sample coordinate may differ by: y1 + ph*bh contracted into one FMA (1), x2 - x1 contracted on the
#                 scaled corner (1, carried into y through ph*bh <= rh), and the final add (1); one more for margin

# ------------------------------------------------------------------ the launch table
# dt_roi_align: (f32, x3_mode, round_tf32, T, P, sampling, levels, n_dev given)
ROI_ALIGN = {
    (0, 0, 0, 1, 7, 2, 4, False), (0, 0, 0, 1, 14, 2, 4, False),      # FPN heads, bf16 (inference and training)
    (0, 2, 0, 1, 7, 2, 4, False), (0, 1, 0, 1, 14, 2, 4, False),      # FPN heads, bf16 pairs: planar FC rows / per position
    (1, 2, 0, 1, 7, 2, 4, False), (1, 1, 0, 1, 14, 2, 4, False),      # FPN heads, tf32 pairs
    (0, 0, 0, 3, 7, 2, 1, False), (0, 0, 0, 3, 14, 2, 1, False),      # tube heads (r18tube), bf16
    (0, 1, 0, 3, 7, 2, 1, False), (0, 1, 0, 3, 14, 2, 1, False),      # tube heads, bf16 pairs
    (1, 1, 0, 3, 7, 2, 1, False), (1, 1, 0, 3, 14, 2, 1, False),      # tube heads, tf32 pairs
}
ROI_ALIGN_BWD = {(1, 7, 2, 4), (1, 14, 2, 4)}                           # (T, P, sampling, levels)
MAXPOOL = {(f32, x3, k, s, p) for (f32, x3) in ((0, 0), (0, 1), (1, 1)) for (k, s, p) in ((3, 2, 1), (1, 2, 0))}
PREP = {(0, (3, 4), 1, False), (3, (3, 4), 1, False), (2, (0, 0), 0, False)}     # (mode, border, row planes, resized)
KP_DECODE = {(1, False, False), (3, False, False)}                     # (T, min_size > 0, heatmaps wanted)
SPATIAL_MEAN = {(0, 0, 0), (0, 1, 0), (1, 1, 0)}                        # (f32, x3, round_tf32)
FOLD = {(3,)}                                                           # (T,)
SCALE_ROIS = {('per_image', 4), ('per_image', 12)}                     # (image index from, ncols)
TABLE = dict(dt_roi_align=ROI_ALIGN, dt_roi_align_bwd=ROI_ALIGN_BWD, dt_maxpool2d=MAXPOOL, dt_prep_clip=PREP,
             dt_keypoint_decode=KP_DECODE, dt_spatial_mean=SPATIAL_MEAN, dt_fold_tube_heads=FOLD, dt_scale_rois=SCALE_ROIS)


def launch_key(name, a):
    """The table key of one L.call(name, *a) of these entry points, or None for other entry points."""
    if name == 'dt_roi_align':
        return (a[8], a[18], a[17], a[13], a[15], a[16], a[4], a[11] is not None)
    if name == 'dt_roi_align_bwd':
        return (a[12], a[14], a[15], a[5])
    if name == 'dt_maxpool2d':
        return (a[9], a[10], a[6], a[7], a[8])
    if name == 'dt_prep_clip':
        return (a[14], (a[11], a[12]), a[13], (a[6], a[7]) != (a[2], a[3]))
    if name == 'dt_keypoint_decode':
        return (a[4], a[9] > 0, a[10] is not None)
    if name == 'dt_spatial_mean':
        return (a[6], a[8], a[7])
    if name == 'dt_fold_tube_heads':
        return (a[3],)
    if name == 'dt_scale_rois':
        return ('batch_idx' if a[4] is not None else 'per_image', a[3])
    return None


def test_step_dense_ops_are_all_in_the_table(record_property):
    """One 800 x 1333 clip of each bench workload through DetectionEngine.detect in bf16, bf16x3, bf16x3h and tf32x3 (the
    last two where the engine takes them), and one KeypointRcnnTrainer.step at the bench training config: every launch of
    the dense entry points has a key in TABLE, each of which has a value test below."""
    import step_launches as sl
    missing, seen = {}, set()
    for run in [(wl, m) for wl in sl.WORKLOADS for m in ('bf16', 'bf16x3', 'bf16x3h', 'tf32x3')] + ['train']:
        rec = sl.record(run)
        tag = run if run == 'train' else '%s_%s' % run
        if not rec.taken:
            assert run[1] not in ('bf16', 'bf16x3'), run
            record_property('not_taken_' + tag, True)
            continue
        launched = [(name, k) for name, a, _ in rec.calls if (k := launch_key(name, a)) is not None]
        record_property('launches_' + tag, len(launched))
        names = {n for n, _ in launched}
        assert {'dt_roi_align_bwd'} <= names if run == 'train' else {'dt_roi_align', 'dt_keypoint_decode'} <= names
        for name, k in launched:
            seen.add((name, k))
            if k not in TABLE[name]:
                missing.setdefault((name, k), run)
    record_property('keys_seen', len(seen))
    assert not missing, missing


# ------------------------------------------------------------------ RoIAlign
IMG_H, IMG_W = 800, 1333
FPN_SHAPES = [(200, 336), (100, 168), (50, 84), (25, 42)]       # P2..P5 of the 800 x 1344 blob
TUBE_SHAPE = (50, 84)                                           # R18 conv4 (stride 16) of the 800 x 1334 blob
C_FEAT = 256


def _store(v, f32, x3):
    """fp32 values -> (device storage rows, the fp32 values they hold)."""
    if x3:
        p = pairs(v, 'tf32' if f32 else 'bf16')
        c = v.shape[-1]
        return p, join(p[..., :c], p[..., c:])
    if f32:
        return v, v
    b = v.bfloat16()
    return b, b.float()


def _crafted_rois(nimg, T, nl):
    """Edge rows (image space), with the level each is routed to: exact fp32 sample grids (7*2^j feature units) whose samples
    land on -1, 0, H-1 and H, RoIs partly and wholly outside the map, and widths / heights below 1 feature unit."""
    rows, lv = [], []
    shapes = FPN_SHAPES if nl == 4 else [TUBE_SHAPE]
    stride = [4, 8, 16, 32] if nl == 4 else [16]
    for li, ((H, W), s) in enumerate(zip(shapes, stride)):
        for b in range(nimg):
            # feature units: bins of 4 (samples at y1 + 4*ph + 1, + 3) from y1 = -2 (first sample at -1) and to H (last)
            for (fx1, fy1, fw, fh) in ((-2, -2, 28, 28), (W - 26, H - 26, 28, 28), (-2, H - 26, 28, 28), (0, 0, 7, 7),
                                       (W - 8, H - 8, 7, 7), (-1, -1, 14, 7), (W + 5, H + 5, 14, 14), (-40, -40, 7, 14),
                                       (3.25, 5.5, 0.5, 0.25), (W / 2, H / 3, 0.75, 3.5)):
                box = [fx1 * s, fy1 * s, (fx1 + fw) * s, (fy1 + fh) * s]
                rows.append([b] + box * T)
                lv.append(li + 2 if nl == 4 else 2)
    return np.array(rows, F32), np.array(lv, np.int32)


def _random_rois(rng, R, nimg, T, dyadic):
    x1, y1 = rng.uniform(0, IMG_W - 20, R), rng.uniform(0, IMG_H - 20, R)
    w, h = rng.uniform(2, 500, R), rng.uniform(2, 400, R)
    if dyadic:            # integer corner, width and height multiples of 7/4: exact sample grids at every level
        x1, y1, w, h = np.floor(x1), np.floor(y1), np.ceil(w / 1.75) * 1.75, np.ceil(h / 1.75) * 1.75
    rois = np.zeros((R, 4 * T + 1), F32)
    rois[:, 0] = rng.integers(0, nimg, R)
    for t in range(T):
        sh = np.round(rng.normal(0, 4, (R, 2))) * (t > 0)
        x2, y2 = np.minimum(x1 + w + sh[:, 0], IMG_W - 1), np.minimum(y1 + h + sh[:, 1], IMG_H - 1)
        rois[:, 1 + 4 * t:5 + 4 * t] = np.stack([x1 + sh[:, 0], y1 + sh[:, 1], x2, y2], 1)
    return rois


def _roi_problem(T, P, nl, seed, sampling=2, nimg=2, R=None):
    """Feature maps at the step's level sizes (two images), R RoIs as the step sizes them, a level with no RoIs."""
    from detectandtrack_b200.ops import rpn_ops
    rng = np.random.default_rng(seed)
    R = R or {7: 1000, 14: 104}[P] * nimg                # box head: RPN_POST_NMS_TOP_N per image; keypoints: detection slots
    cr, cl = _crafted_rois(nimg, T, nl)
    rois = np.concatenate([cr, _random_rois(rng, (R - len(cr)) // 2, nimg, T, True),
                           _random_rois(rng, R - len(cr) - (R - len(cr)) // 2, nimg, T, False)])
    if nl == 4:
        lv, _, _ = rpn_ops.distribute(torch.from_numpy(rois).cuda(), None, col0=1, T=1, want_restore=False)
        lv = lv.cpu().numpy().copy()
        lv[:len(cr)] = cl
        lv[lv == 5] = 4                                                 # P5 gets no RoI
        shapes = FPN_SHAPES
    else:
        lv, shapes = None, [TUBE_SHAPE]
    return rois, lv, shapes, R


def _roi_tol(A, S, absF, ref, storage, device):
    """Forward bound: each of the 4*gh*gw terms of a bin carries <= 3 roundings (1 - ly, the weight product, the product
    inside the FMA chain), the 4*gh*gw - 1 additions one each and the division by the count one: (4*gh*gw + 3)u, +1 for
    second-order terms, times |S| @ |F|; plus the coordinate term (RoiAlignMatrix.coord_fwd) and the storage rounding of the
    stored value, storage * (|ref| + the above)."""
    n = torch.from_numpy(A.count).to(device)[:, None]
    acc = (4 * n + 4) * U24 * (S @ absF) + A.coord_fwd(absF, K_COORD, device)
    return acc + storage * (ref.abs() + acc)


# (f32, x3 mode, round_tf32) -> relative rounding of the stored value: round-to-nearest to p significant bits is off by at most
# 2^-p |v| (bf16 p = 8, tf32 p = 11); a pair rounds the remainder v - hi (<= 2^-p |v|) once more: 2^-2p
STORAGE = {(0, 0, 0): 2.0 ** -8, (1, 0, 0): 0.0, (1, 0, 1): 2.0 ** -11, (0, 1, 0): 2.0 ** -16, (0, 2, 0): 2.0 ** -16,
           (1, 1, 0): 2.0 ** -22, (1, 2, 0): 2.0 ** -22}

ROI_VALUE_KEYS = sorted(ROI_ALIGN) + [
    (0, 0, 0, 1, 7, 2, 4, True), (0, 1, 0, 1, 14, 2, 4, True), (0, 2, 0, 1, 7, 2, 4, True), (1, 2, 0, 1, 7, 2, 4, True),
    (0, 1, 0, 3, 14, 2, 1, True), (1, 0, 0, 1, 7, 2, 4, False), (1, 0, 1, 1, 7, 2, 4, False),
    (0, 1, 0, 1, 14, 0, 4, False), (0, 1, 0, 3, 7, 0, 1, False), (1, 2, 0, 1, 7, 0, 4, False)]


@pytest.mark.parametrize('key', ROI_VALUE_KEYS, ids=lambda k: '-'.join(str(int(v)) for v in k))
def test_roi_align_step_shape_vs_fp64(key, record_property):
    """dt_roi_align at the step's level sizes, R and C, two images, against S @ F in fp64 on the device.  Sampling 0 checks
    a fixed subset of rows plus every crafted row (its sample grids grow with the RoI); n_dev < R rows must be zero in every
    output mode, the planar lo block included."""
    from detectandtrack_b200.ops import dense_ops
    f32, x3m, rnd, T, P, samp, nl, ndev = key
    rois, lv, shapes, R = _roi_problem(T, P, nl, seed=hash(key) % 1000, sampling=samp)
    g = torch.Generator(device='cuda').manual_seed(11)
    vals = [torch.randn((2 * T, H, W, C_FEAT), generator=g, device='cuda') for H, W in shapes]
    st = [_store(v, f32, x3m) for v in vals]
    n = R - 37 if ndev else R
    n_dev = torch.tensor([n], dtype=torch.int32, device='cuda') if ndev else None
    out = dense_ops.roi_align([s for s, _ in st], [1.0 / 2 ** (2 + i) for i in range(nl)] if nl == 4 else [1 / 16.],
                              torch.from_numpy(rois).cuda(), None if lv is None else torch.from_numpy(lv).cuda(), P, samp,
                              T=T, n_dev=n_dev, round_tf32=bool(rnd), x3_mode=x3m)
    C = C_FEAT
    if x3m == 1:
        hi, lo = out[..., :C], out[..., C:]
    elif x3m == 2:
        blk = T * P * P * C
        hi, lo = out[:, :blk].reshape(R, T, P, P, C), out[:, blk:].reshape(R, T, P, P, C)
    else:
        hi, lo = out, None
    got = join(hi, lo) if lo is not None else hi.float()
    if ndev:                                                        # dead rows: exact zeros, both halves, every layout
        assert torch.equal(out[n:], torch.zeros_like(out[n:]))
    rows = np.arange(n)
    if samp == 0:
        rows = np.unique(np.concatenate([np.arange(min(n, 80)), np.arange(0, n, max(1, n // 120))]))
    A = RoiAlignMatrix([(2 * T, H, W) for H, W in shapes], [1.0 / 2 ** (2 + i) for i in range(nl)] if nl == 4 else [1 / 16.],
                       rois, lv, P, samp, T=T, rows=rows)
    S = A.S('cuda')
    Fm = A.flat([v for _, v in st])
    ref = (S @ Fm).view(len(rows), T, P, P, C)
    tol = _roi_tol(A, S, Fm.abs(), ref.reshape(-1, C), STORAGE[(f32, x3m, rnd)], 'cuda').view(ref.shape)
    err = (got[torch.from_numpy(rows).cuda()].double() - ref).abs()
    record_property('worst_err_over_tol', float((err / tol.clamp_min(1e-300)).max()))
    record_property('exact_rows', int((A.ulp == 0).sum()) // (P * P))
    bad = (err > tol).nonzero()
    assert len(bad) == 0, (len(bad), bad[:5].tolist(), float(err.max()))
    # the crafted exact-grid rows (the first 8 of each 10) carry no coordinate term: their bound is the arithmetic alone
    ncr = 20 * (4 if nl == 4 else 1)
    for i in range(ncr):
        if i % 10 < 8:
            assert (A.ulp[i * T * P * P:(i + 1) * T * P * P] == 0).all(), i


@pytest.mark.parametrize('key', sorted(ROI_ALIGN_BWD), ids=lambda k: '-'.join(map(str, k)))
def test_roi_align_bwd_step_shape_vs_fp64(key, record_property):
    """dt_roi_align_bwd at the training step's shapes (2 x 512 box RoIs at P = 7, 2 x 128 keypoint RoIs at P = 14, C = 256,
    four levels): S^T @ G in fp64, with a cluster of RoIs over the same pixels, and n_dev rows that must scatter nothing.
    Bound: a term v * (hy*hx*inv_cnt) carries <= 4 roundings (1 - ly, two products, the product with v) and the m additions of
    an element's m contributions one each: (m + 4)u, +1 for second-order terms, times |S|^T @ |G|; the atomic order is free.
    Plus the coordinate term (RoiAlignMatrix.coord_bwd)."""
    from detectandtrack_b200 import _lib as L
    from detectandtrack_b200.ops import train_ops as to
    T, P, samp, nl = key
    R = {7: 1024, 14: 256}[P]
    rois, lv, shapes, _ = _roi_problem(T, P, nl, seed=P, nimg=2, R=R)
    rng = np.random.default_rng(4)
    c0 = rng.uniform(300, 500, 2)
    for i in range(60, 260 if R > 300 else 120):                          # many RoIs over the same pixels of P3
        rois[i, 0] = 1
        rois[i, 1:5] = [c0[0] + rng.normal(0, 2), c0[1] + rng.normal(0, 2), c0[0] + 150 + rng.normal(0, 2), c0[1] + 200 + rng.normal(0, 2)]
        lv[i] = 3
    g = torch.Generator(device='cuda').manual_seed(12)
    G = torch.randn((R, T, P, P, C_FEAT), generator=g, device='cuda').bfloat16()
    scales = [1.0 / 2 ** (2 + i) for i in range(nl)]
    rois_d, lv_d = torch.from_numpy(rois).cuda(), torch.from_numpy(lv).cuda()
    A = RoiAlignMatrix([(2 * T, H, W) for H, W in shapes], scales, rois, lv, P, samp, T=T)
    S = A.S('cuda')
    for n in (R, R - 29):
        dfe = [L.zeros((2 * T, H, W, C_FEAT), torch.float32) for H, W in shapes]
        to.roi_align_bwd(G, dfe, scales, rois_d, lv_d, P, samp, T=T,
                         n_dev=None if n == R else torch.tensor([n], dtype=torch.int32, device='cuda'))
        Gd = G.double().reshape(-1, C_FEAT).clone()
        Gd[n * T * P * P:] = 0                                            # rows past n_dev scatter nothing
        ref = S.t() @ Gd
        m = torch.from_numpy(A.col_terms).cuda().double()[:, None]
        tol = (m + 5) * U24 * (S.t() @ Gd.abs()) + A.coord_bwd(Gd.abs(), K_COORD, 'cuda')
        got = A.flat(dfe)
        err = (got - ref).abs()
        record_property('worst_err_over_tol_n%d' % n, float((err / tol.clamp_min(1e-300)).max()))
        record_property('max_terms', int(A.col_terms.max()))
        bad = (err > tol).nonzero()
        assert len(bad) == 0, (n, len(bad), bad[:5].tolist(), float(err.max()))


# ------------------------------------------------------------------ keypoint decode
S_KP, K_KP = 14, 17


def _seam_box(profile, n_src, seam):
    """The smallest output size >= seam + 1 whose cubic resize of `profile` (fp64, length n_src) peaks exactly at index
    `seam` with a margin, so the maximum lies on a strip / row-block seam."""
    for d in range(seam + 1, 1400):
        v = cubic_matrix(d, n_src) @ profile
        top = v.topk(2).values
        if int(v.argmax()) == seam and float(top[0] - top[1]) > 1e-3 * float(top[0]):
            return d
    raise AssertionError('no seam size')


def _kp_problem(T, D, seed):
    """lowres [D*T, S, S, 68] (sub-pixel packed, frame t of detection d at row d*T + t), boxes [D, 4T + 1]: crafted rows
    (1333 x 800, 257 x 300, 512 x 513, a zero-size dead slot, a flat map, a maximum on the strip and row-block seam) then
    random boxes; per-frame boxes differ."""
    rng = np.random.default_rng(seed)
    g = torch.Generator().manual_seed(seed)
    low = torch.nn.functional.avg_pool2d(torch.randn((D * T, K_KP, 2 * S_KP, 2 * S_KP), generator=g), 3, 1, 1) * 3
    boxes = np.zeros((D, 4 * T + 1), F32)
    x1, y1 = rng.uniform(0, 1000, D), rng.uniform(0, 500, D)
    w, h = rng.uniform(1, 333, D), rng.uniform(1, 300, D)
    for t in range(T):
        sh = rng.normal(0, 3, (D, 4)) * (t > 0)
        boxes[:, 4 * t:4 * t + 4] = np.stack([x1, y1, x1 + w, y1 + h], 1) + sh
    crafted = [(0, 0, 1333, 800), (10.5, 20.25, 267.5, 320.25), (100, 50, 612, 563), (0, 0, 0, 0), (40, 30, 340, 320)]
    for d, b in enumerate(crafted):
        boxes[d, :4 * T] = np.tile(np.array(b, F32), T) + np.repeat(np.arange(T, dtype=F32), 4) * 2 * (d != 3)
    low[4 * T:5 * T] = 0                                                # flat map: the tie goes to index 0
    # maximum on the seam: a separable non-negative bump whose resize peaks at column 256 and row 256
    a = torch.zeros(2 * S_KP); a[9], a[10] = 100.0, 30.0
    U = upsample2x_matrix(2 * S_KP)
    wsz = _seam_box(U @ a.double(), 4 * S_KP, 256)
    for t in range(T):
        low[5 * T + t] = (a[:, None] * a[None, :])[None].float()
        boxes[5, 4 * t:4 * t + 4] = [7.0 + t, 9.0, 7.0 + t + wsz, 9.0 + wsz]
    packed = low.view(D * T, K_KP, S_KP, 2, S_KP, 2).permute(0, 2, 4, 3, 5, 1).reshape(D * T, S_KP, S_KP, 4 * K_KP)
    ld = 68
    lowp = torch.zeros((D * T, S_KP, S_KP, ld))
    lowp[..., :4 * K_KP] = packed
    return lowp, low, boxes, 6


def _prob_rel_tol(rw, rh, rng_val, e_max):
    """The probability's relative bound: a thread sums n_t terms sequentially (n_t from the kernel's strip / row-phase split:
    256 threads, strips of 256 columns, 4 columns per thread), then a 5-level shuffle tree and 8 warps: (n_t + 16)u; __expf has
    relative error (2 + 1.16|x|) * 2^-23 per term and per rescale of the running sum (the rescales' |x| add up to at most the
    map's range); the logits themselves are off by <= e_max each, so a term's exponent by <= 2 e_max."""
    n_t = 0
    for x0 in range(0, rw, 256):
        sw = min(256, rw - x0)
        nseg = max(1, 256 // ((sw + 3) // 4))
        n_t += 4 * -(-rh // nseg)
    return (n_t + 16) * U24 + 2.0 ** -23 * (2 * n_t + 2 + 2.32 * rng_val) + 4.1 * e_max


KP_VALUE_KEYS = sorted(KP_DECODE) + [(1, True, True), (3, True, True), (1, False, True)]


@pytest.mark.parametrize('key', KP_VALUE_KEYS, ids=lambda k: '-'.join(str(int(v)) for v in k))
def test_keypoint_decode_step_shape_vs_fp64(key, record_property):
    """dt_keypoint_decode over the step's D = 104 detection slots of one clip, K = 17, 56 x 56 maps, boxes in image space,
    against the fp64 upsample, Ry @ M @ Rx^T and heatmaps_to_keypoints, on every crafted row and a fixed subset of the rest.
    Map bound: the 2x upsample has <= 4 terms of exact weights (1/16, 3/16, 9/16): 4u |.|; the cubic passes add 4 + 4 terms
    (16u with the input's) and the fp32 cubic coefficients may differ from cv2's fp32 order by contraction: each of c0..c2 by
    <= 2^-16 (8 operations on values <= 12), c3 by 3x that, summed over two passes of weights <= 1.3: 2^-12 max|heat|."""
    from detectandtrack_b200.ops import dense_ops
    T, has_min, want_heat = key
    min_size = 100 if has_min else 0
    D = 104
    lowp, low, boxes, ncrafted = _kp_problem(T, D, seed=T + 2 * has_min)
    bx = torch.from_numpy(boxes).cuda()
    xy, heat = dense_ops.keypoint_decode(lowp.cuda(), bx, K_KP, T, min_size=min_size, want_heatmaps=want_heat)
    xy = xy.cpu().numpy()
    check = list(range(ncrafted)) + list(range(ncrafted, D, 4))
    worst = 0.0
    for d in check:
        for t in range(T):
            lo = low[d * T + t].cuda()
            hmap, res, resabs, geo = keypoint_maps_ref(lo, boxes[d, 4 * t:4 * t + 4], min_size)
            rw, rh, wc, hc, ox, oy = geo
            if want_heat:
                Uu = upsample2x_matrix(2 * S_KP).cuda()
                htol = 4 * U24 * (Uu @ lo.double().abs() @ Uu.t())
                assert ((heat[d, t * K_KP:(t + 1) * K_KP].double() - hmap).abs() <= htol).all(), (d, t)
            hmax = hmap.abs().flatten(1).max(1).values[:, None, None]
            tol = 16 * U24 * resabs + 2.0 ** -12 * hmax                     # [K, rh, rw]
            ref_xy, ref_pos = keypoints_from_maps(res, geo)
            flat, tflat = res.flatten(1), tol.flatten(1)
            for k in range(K_KP):
                col = t * K_KP + k
                # the device (x, y) must be fp32((x_int + 0.5) * wcorr + offset) of integer pixels, computed that way
                xs = ((np.arange(rw) + 0.5) * np.float64(wc) + np.float64(ox)).astype(F32)
                ys = ((np.arange(rh) + 0.5) * np.float64(hc) + np.float64(oy)).astype(F32)
                xi, yi = np.where(xs == xy[d, 0, col])[0], np.where(ys == xy[d, 1, col])[0]
                assert len(xi) >= 1 and len(yi) >= 1, (d, t, k)
                xi, yi = int(xi[0]), int(yi[0])
                p, rp = yi * rw + xi, int(ref_pos[k])
                mx, tmax = flat[k, rp].item(), tflat[k].max().item()
                # the chosen pixel's fp64 value is within the two pixels' bounds of the fp64 maximum
                assert flat[k, p].item() >= mx - tflat[k, p].item() - tflat[k, rp].item(), (d, t, k, p, rp)
                # a clear fp64 winner (beats every other pixel by more than twice the bound) must be chosen
                second = flat[k].clone(); second[rp] = -np.inf
                if mx - second.max().item() > 2 * tmax:
                    assert p == rp, (d, t, k, p, rp)
                    assert xy[d, 0, col] == F32(ref_xy[0, k]) and xy[d, 1, col] == F32(ref_xy[1, k])
                assert abs(xy[d, 2, col] - mx) <= 2 * tmax, (d, t, k)
                rel = _prob_rel_tol(rw, rh, mx - flat[k].min().item(), tmax)
                assert abs(xy[d, 3, col] - ref_xy[3, k]) <= rel * ref_xy[3, k], (d, t, k, xy[d, 3, col], ref_xy[3, k])
                worst = max(worst, abs(xy[d, 2, col] - mx) / (2 * tmax))
                if d == 4:                                                   # flat map: first index, 1 / (rw * rh)
                    assert p == 0 and abs(xy[d, 3, col] * rw * rh - 1) <= rel, (d, t, k, p)
                if d == 5 and k == 0:                                        # the maximum on the seam (column and row 256)
                    assert (xi, yi) == (256, 256), (xi, yi)
    record_property('worst_logit_err_over_tol', worst)


# ------------------------------------------------------------------ max-pool
MAXPOOL_SHAPES = {(3, 2, 1): [(3, 400, 672, 64), (3, 25, 41, 64)], (1, 2, 0): [(3, 25, 42, 256), (3, 25, 41, 256)]}


@pytest.mark.parametrize('key', sorted(MAXPOOL), ids=lambda k: '-'.join(map(str, k)))
def test_maxpool_step_shape_bit_exact(key):
    """pool1 (3x3 s2 p1, the rolling-row kernel) on conv1's [B*T, 400, 672, 64] output and P6 (1x1 s2) on the frames-outermost
    [T*B, 25, 42, 256] P5 stack, plus odd widths: bit-exact.  The max is exact, and re-splitting a canonical pair returns it."""
    from detectandtrack_b200.ops import dense_ops
    f32, x3, k, s, p = key
    g = torch.Generator(device='cuda').manual_seed(13)
    for shp in MAXPOOL_SHAPES[(k, s, p)]:
        v = torch.randn(shp, generator=g, device='cuda') * 3
        v[:, :, :, :8] = v[:, :, :1, :8]                     # equal values along a row: ties
        if x3:
            x = pairs(v, 'tf32' if f32 else 'bf16')
            vv = join(x[..., :shp[-1]], x[..., shp[-1]:])
            exp = pairs(maxpool_ref(vv, k, s, p).float(), 'tf32' if f32 else 'bf16')
        else:
            x = v if f32 else v.bfloat16()
            exp = maxpool_ref(x, k, s, p).to(x.dtype)
        y = dense_ops.maxpool2d(x.contiguous(), k, s, p, x3=bool(x3))
        assert y.shape == exp.shape and torch.equal(y, exp), shp


# ------------------------------------------------------------------ blob prep
PREP_VALUE_KEYS = sorted(PREP, key=str) + [(3, (3, 4), 1, True), (0, (3, 4), 1, True), (2, (0, 0), 0, True)]


@pytest.mark.parametrize('key', PREP_VALUE_KEYS, ids=lambda k: '%d-%d%d-%d-%d' % (k[0], k[1][0], k[1][1], k[2], k[3]))
def test_prep_clip_step_shape(key):
    """dt_prep_clip on an 800 x 1333 clip at scale 1 (bit-exact: the hi half is bf16(p - mean), the lo half bf16(v - hi)) and a
    720 x 1280 PoseTrack-sized clip resized by 1333/1280 to 750 x 1333 (bound: two 2-term passes with exact weights 1 - f, f:
    4u, +1 second order, times the resize of |p - mean|, then the storage rounding), with the border and row planes."""
    from detectandtrack_b200.ops import dense_ops
    from detectandtrack_b200.modeling.engine import im_scale_and_size, padded_blob_size
    mode, (by, bx), planes, resized = key
    H, W = (720, 1280) if resized else (800, 1333)
    scale, (hr, wr) = im_scale_and_size(H, W, 800, 1333)
    hp, wp = padded_blob_size([(hr, wr)], 32.0)
    hp, wp = hp + (hp & 1), wp + (wp & 1)
    assert resized == ((hr, wr) != (H, W))
    means = np.array([102.9801, 115.9465, 122.7717], F32)
    rng = np.random.default_rng(14)
    fr = rng.integers(0, 256, (3, H, W, 3), dtype=np.uint8)
    cpad = 4 if mode == 2 else 8
    out = dense_ops.prep_clip(torch.from_numpy(fr).cuda(), means, scale, (hr, wr), (hp, wp), cpad=cpad, out_f32=mode,
                              border=(by, bx), row_planes=bool(planes)).cpu()
    Ht, Wt = hp + 2 * by, wp + 2 * bx
    if planes:                                                           # padded row r lives at [r & 1][r >> 1]
        full = torch.empty((3, Ht, Wt, cpad), dtype=out.dtype)
        full[:, 0::2], full[:, 1::2] = out[:, 0], out[:, 1]
        out = full
    assert torch.equal(out[:, :by], torch.zeros_like(out[:, :by])) and torch.equal(out[:, Ht - by:], torch.zeros_like(out[:, Ht - by:]))
    assert torch.equal(out[:, :, :bx], torch.zeros_like(out[:, :, :bx])) and torch.equal(out[:, :, Wt - bx:], torch.zeros_like(out[:, :, Wt - bx:]))
    core = out[:, by:by + hp, bx:bx + wp]
    if mode == 3:
        hi, lo = core[..., :3], core[..., 3:6]
        assert torch.equal(core[..., 6:], torch.zeros_like(core[..., 6:]))
        got = join(hi, lo)
    else:
        got = core[..., :3].float()
        assert torch.equal(core[..., 3:], torch.zeros_like(core[..., 3:]))
    ref = prep_ref(fr, means, scale, (hr, wr), (hp, wp))
    if not resized:
        v = ref.float()                                                  # (float)p - mean: one fp32 rounding, as the kernel
        if mode == 3:
            eh, el = split_bf16(v)
            assert torch.equal(hi, eh) and torch.equal(lo, el)
        else:
            assert torch.equal(got, v if mode == 2 else v.bfloat16().float())
        return
    storage = {3: 2.0 ** -16, 0: 2.0 ** -8, 2: 0.0}[mode]       # see STORAGE
    A = torch.zeros_like(ref)
    for f in range(3):
        A[f, :hr, :wr] = linear_abs(fr[f].astype(F32) - means, (hr, wr), scale)
    acc = 5 * U24 * A
    tol = acc + storage * (ref.abs() + acc)
    assert ((got.double() - ref).abs() <= tol).all(), float((got.double() - ref).abs().max())


# ------------------------------------------------------------------ 3-D box head glue
@pytest.mark.parametrize('key', sorted(SPATIAL_MEAN) + [(1, 0, 0), (1, 0, 1)], ids=lambda k: '-'.join(map(str, k)))
def test_spatial_mean_step_shape_bit_exact(key):
    """The r18tube box head's mean over the 4 x 4 res5 output of 1000 tubes x 3 frames, C = 512: bit-exact against the
    sequential fp32 restatement (per row a sum over W, / W, rows summed, / H), then the storage's rounding or split."""
    from detectandtrack_b200.ops import dense_ops
    f32, x3, rnd = key
    g = torch.Generator().manual_seed(15)
    v = torch.randn((3000, 4, 4, 512), generator=g)
    if x3:
        kind = 'tf32' if f32 else 'bf16'
        x = pairs(v, kind)
        ref = pairs(spatial_mean_seq(join(x[..., :512], x[..., 512:])), kind)
    elif f32:
        x = v
        m = spatial_mean_seq(x)
        ref = round_tf32(m) if rnd else m
    else:
        x = v.bfloat16()
        ref = spatial_mean_seq(x).bfloat16()
    y = dense_ops.spatial_mean(x.cuda(), round_tf32=bool(rnd), x3=bool(x3)).cpu()
    assert torch.equal(y, ref)


def test_fold_tube_heads_step_shape_bit_exact():
    """[R*T, ld] per-frame [cls | bbox] of 1000 tubes x 3 frames, 2 classes, the engine's row stride: cls = sequential fp32
    mean over t, bbox re-ordered to channel c*4T + 4t + k: bit-exact."""
    from detectandtrack_b200.ops import dense_ops
    g = torch.Generator().manual_seed(16)
    R, T, C, ld = 1000, 3, 2, 12
    o = torch.randn((R * T, ld), generator=g)
    cls, bbox = dense_ops.fold_tube_heads(o.cuda(), R, T, C)
    ec, eb = fold_tube_heads_ref(o, R, T, C)
    assert torch.equal(cls.cpu(), ec) and torch.equal(bbox.cpu(), eb)


@pytest.mark.parametrize('how', ['per_image', 'batch_idx'])
@pytest.mark.parametrize('ncols', [4, 12])
def test_scale_rois_bit_exact(how, ncols):
    """Keypoint RoIs from the detection slots (row stride 4T + 1, 104 slots per clip, two clips): fp64 product, then fp32; the
    image index from the slot (i // per_image) or a batch_idx column."""
    from detectandtrack_b200.ops import dense_ops
    g = torch.Generator().manual_seed(17)
    D = 208
    dets = torch.rand((D, ncols + 1), generator=g) * 1333
    bidx = (torch.arange(D) % 2).float()
    scale = 1333 / 1280
    kw = dict(batch_idx=bidx.cuda()) if how == 'batch_idx' else dict(per_image=104)
    got = dense_ops.scale_rois(dets.cuda(), ncols, scale, **kw).cpu()
    exp = scale_rois_ref(dets, ncols, scale, **({'batch_idx': bidx} if how == 'batch_idx' else {'per_image': 104}))
    assert torch.equal(got, exp)
