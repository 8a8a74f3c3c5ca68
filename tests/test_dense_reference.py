"""CPU: the fp64 references the dense-op value tests (tests/test_gpu_dense_step.py) compare csrc/dense_ops.cu and the RoIAlign
backward of csrc/train_ops.cu with.  They are written from the operators' documented semantics (Caffe2 RoIAlign with
aligned=False, cv2 INTER_LINEAR / INTER_CUBIC, heatmaps_to_keypoints), share no code with the kernels, and run as torch
float64 on either device.  Where the operator's own arithmetic decides something discrete (RoIAlign sample positions and
clamps, cv2's resize coefficients) that part is done in fp32 as the operator does it, and only the sums are fp64.
Each reference is pinned here once against an independent implementation on small shapes."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

F32 = np.float32
U24 = 2.0 ** -24                  # unit roundoff of fp32


# ------------------------------------------------------------------ split storage
def split_bf16(v):
    """fp32 tensor -> (hi, lo) bf16 with hi = bf16(v), lo = bf16(v - hi)."""
    v = v.float()
    hi = v.bfloat16()
    return hi, (v - hi.float()).bfloat16()


def round_tf32(v):
    """fp32 -> nearest tf32 (10 explicit mantissa bits), ties to even, as fp32."""
    u = v.float().contiguous().view(torch.int32).long() & 0xFFFFFFFF
    u = (u + 0xFFF + ((u >> 13) & 1)) & 0xFFFFE000
    return u.to(torch.int64).where(u < 2 ** 31, u - 2 ** 32).to(torch.int32).view(torch.float32)


def split_tf32(v):
    v = v.float()
    hi = round_tf32(v)
    return hi, round_tf32(v - hi)


def join(hi, lo):
    return hi.float() + lo.float()


def pairs(v, kind):
    """fp32 [..., C] -> [..., 2C] pair rows [hi | lo] of `kind` 'bf16' or 'tf32'."""
    hi, lo = split_bf16(v) if kind == 'bf16' else split_tf32(v)
    return torch.cat([hi, lo], -1)


# ------------------------------------------------------------------ RoIAlign as a sparse sample matrix
class RoiAlignMatrix:
    """Caffe2 RoIAlign (aligned=False) of RoIs `rois` [R, 4T+1] over per-level maps of shapes `level_shapes`
    [(N_l, H_l, W_l)] as one sparse fp64 matrix S: output row ((i*T + t)*P + ph)*P + pw (i indexes `rows`) x
    feature column off_l + (img*H_l + y)*W_l + x, img = rois[r, 0]*T + t, level levels[r] - k_min.  Forward = S @ F,
    backward = S^T @ G for F the levels' [N*H*W, C] maps concatenated.

    The geometry (scaled box, max(., 1), bin sizes, sample grid, validity window, clamps, bilinear weights) is fp32 in
    Caffe2's order; the 1 / count is applied in fp64.  `ulp` [rows*T] is 0 for RoIs whose every geometry step is exact in
    fp32 (then any FMA contraction computes the same samples) and otherwise ulp(max |scaled corner| + 1)."""

    def __init__(self, level_shapes, scales, rois, levels, P, sampling, T=1, k_min=2, rows=None):
        rois = np.asarray(rois, F32)
        R = rois.shape[0]
        rows = np.arange(R) if rows is None else np.asarray(rows, np.int64)
        lv = np.zeros(R, np.int64) if levels is None else np.asarray(levels, np.int64) - k_min
        self.offs = np.cumsum([0] + [n * h * w for n, h, w in level_shapes])
        self.level_shapes, self.P, self.T, self.nrows = level_shapes, P, T, len(rows) * T * P * P
        Hs, Ws = np.array([s[1] for s in level_shapes]), np.array([s[2] for s in level_shapes])
        scl = np.asarray(scales, F32)
        ri, ci, wi, cnt_row, ulp_row = [], [], [], np.zeros(len(rows) * T), np.zeros(len(rows) * T)
        for t in range(T):
            ro, l = rois[rows], lv[rows]
            sc, H, W = scl[l], Hs[l], Ws[l]
            img = ro[:, 0].astype(np.int64) * T + t
            c = [ro[:, 1 + 4 * t + j] * sc for j in range(4)]
            x1, y1, x2, y2 = c
            exact = np.ones(len(rows), bool)

            def ex(v32, v64):
                nonlocal exact
                exact &= v32.astype(np.float64) == v64
                return v32
            for j in range(4):
                ex(c[j], ro[:, 1 + 4 * t + j].astype(np.float64) * sc.astype(np.float64))
            rw = np.maximum(ex(x2 - x1, x2.astype(np.float64) - x1), F32(1))
            rh = np.maximum(ex(y2 - y1, y2.astype(np.float64) - y1), F32(1))
            bh, bw = ex(rh / F32(P), rh / np.float64(P)), ex(rw / F32(P), rw / np.float64(P))
            if sampling > 0:
                gh = gw = np.full(len(rows), sampling, np.int64)
            else:
                gh, gw = np.ceil(rh / F32(P)).astype(np.int64), np.ceil(rw / F32(P)).astype(np.int64)
            m = np.max(np.abs(np.stack(c)), 0).astype(F32) + F32(1)
            for g in sorted(set(zip(gh.tolist(), gw.tolist()))):
                sel = np.where((gh == g[0]) & (gw == g[1]))[0]
                gy, gx = g
                pp = np.arange(P, dtype=F32)

                def coords(a1, b, gn):
                    base = a1[sel, None] + pp[None, :] * b[sel, None]                       # [n, P]
                    off = (np.arange(gn, dtype=F32) + F32(0.5))[None, :] * b[sel, None] / F32(gn)    # [n, g]
                    ok = (a1[sel, None].astype(np.float64) + pp[None, :].astype(np.float64) * b[sel, None] == base).all(1)
                    ok &= ((np.arange(gn) + 0.5)[None, :] * b[sel, None].astype(np.float64) / gn == off).all(1)
                    s = base[:, :, None] + off[:, None, :]                                   # [n, P, g]
                    ok &= (base[:, :, None].astype(np.float64) + off[:, None, :] == s).all((1, 2))
                    return s, ok
                ys, oky = coords(y1, bh, gy)
                xs, okx = coords(x1, bw, gx)
                exact[sel] &= oky & okx
                n = len(sel)
                y = np.broadcast_to(ys[:, :, None, :, None], (n, P, P, gy, gx)).copy()       # [n, ph, pw, iy, ix]
                x = np.broadcast_to(xs[:, None, :, None, :], (n, P, P, gy, gx)).copy()
                Hn = np.broadcast_to(H[sel, None, None, None, None], y.shape)
                Wn = np.broadcast_to(W[sel, None, None, None, None], y.shape)
                valid = (y >= -1) & (y <= Hn) & (x >= -1) & (x <= Wn)
                y, x = np.maximum(y, F32(0)), np.maximum(x, F32(0))
                yl, xl = y.astype(np.int64), x.astype(np.int64)
                ytop, xtop = yl >= Hn - 1, xl >= Wn - 1
                yl, xl = np.where(ytop, Hn - 1, yl), np.where(xtop, Wn - 1, xl)
                yh, xh = np.where(ytop, yl, yl + 1), np.where(xtop, xl, xl + 1)
                y, x = np.where(ytop, yl.astype(F32), y), np.where(xtop, xl.astype(F32), x)
                ly, lx = y - yl.astype(F32), x - xl.astype(F32)
                hy, hx = F32(1) - ly, F32(1) - lx
                base_col = self.offs[l[sel]][:, None, None, None, None] + img[sel][:, None, None, None, None] * (Hn * Wn)
                row = (((sel[:, None, None, None, None] * T + t) * P + np.arange(P)[None, :, None, None, None]) * P
                       + np.arange(P)[None, None, :, None, None])
                row = np.broadcast_to(row, y.shape)
                for yy, xx, w in ((yl, xl, hy * hx), (yl, xh, hy * lx), (yh, xl, ly * hx), (yh, xh, ly * lx)):
                    ri.append(row[valid]); ci.append((base_col + yy * Wn + xx)[valid])
                    wi.append(w[valid].astype(np.float64) / (gy * gx))
                cnt_row[sel * T + t] = gy * gx
            ulp_row[np.arange(len(rows)) * T + t] = np.where(exact, 0.0, np.spacing(m).astype(np.float64))
        self.rows_i = np.concatenate(ri) if ri else np.zeros(0, np.int64)
        self.cols_i = np.concatenate(ci) if ci else np.zeros(0, np.int64)
        self.w = np.concatenate(wi) if wi else np.zeros(0)
        self.ncols = int(self.offs[-1])
        self.count = np.repeat(cnt_row, P * P)            # gh*gw of each output row
        self.ulp = np.repeat(ulp_row, P * P)              # per output row
        self.col_terms = np.bincount(self.cols_i, minlength=self.ncols)     # contributions to each feature element

    def _sparse(self, vals, device):
        idx = torch.from_numpy(np.stack([self.rows_i, self.cols_i]))
        s = torch.sparse_coo_tensor(idx, torch.from_numpy(vals), (self.nrows, self.ncols), dtype=torch.float64)
        return s.coalesce().to(device)

    def S(self, device='cpu'):
        return self._sparse(self.w, device)

    def U(self, k, device='cpu'):
        """Coordinate-error weights: 2k*ulp / count on every (sample, corner) entry (see coord_fwd / coord_bwd)."""
        return self._sparse(2.0 * k * self.ulp[self.rows_i] / self.count[self.rows_i], device)

    def flat(self, maps):
        """per-level [N, H, W, C] -> [ncols, C] fp64 (the matrix's column order)."""
        return torch.cat([m.double().reshape(-1, m.shape[-1]) for m in maps], 0)

    def unflat(self, x):
        return [x[self.offs[i]:self.offs[i + 1]].view(n, h, w, -1) for i, (n, h, w) in enumerate(self.level_shapes)]

    def sumpool3(self, x):
        """[ncols, C] -> the 3x3 neighbourhood sum per level map (zero outside)."""
        out = []
        for m in self.unflat(x):
            p = F.pad(m, (0, 0, 1, 1, 1, 1))
            out.append(sum(p[:, dy:dy + m.shape[1], dx:dx + m.shape[2]] for dy in range(3) for dx in range(3)))
        return self.flat(out)

    def coord_fwd(self, absF, k, device='cpu'):
        """A sample coordinate that differs by at most k ulps (nvcc contracts y1 + ph*bh + ... into FMAs) moves each bilinear
        weight by at most 2k*ulp (|dw/dy|, |dw/dx| <= 1), also when the sample crosses into a neighbouring cell, whose
        corners lie in the 3x3 neighbourhood of the old ones: |error| <= U @ sumpool3(|F|)."""
        return self.U(k, device) @ self.sumpool3(absF)

    def coord_bwd(self, absG, k, device='cpu'):
        """The same moved weight mass, scattered: |error| <= sumpool3(U^T @ |G|)."""
        return self.sumpool3(self.U(k, device).t() @ absG)


def roi_align_ref(maps, scales, rois, levels, P, sampling, T=1, k_min=2, rows=None):
    """maps: per-level [N, H, W, C] (any float type) -> fp64 [len(rows), T, P, P, C] and the matrix."""
    A = RoiAlignMatrix([tuple(m.shape[:3]) for m in maps], scales, rois, levels, P, sampling, T, k_min, rows)
    y = A.S(maps[0].device) @ A.flat(maps)
    return y.view(-1, T, P, P, maps[0].shape[-1]), A


# ------------------------------------------------------------------ blob prep
def linear_coeffs(dst, src, inv_scale):
    """cv2 INTER_LINEAR source index and fp32 weight of each destination index: f = (float)((d + 0.5) / scale - 0.5),
    s = floor(f), clamped to [0, src - 1] (weight 0 on the far sample at the borders)."""
    f = ((np.arange(dst) + 0.5) * inv_scale - 0.5).astype(F32)
    s = np.floor(f).astype(np.int64)
    f = f - s.astype(F32)
    f = np.where(s < 0, F32(0), f)
    s = np.maximum(s, 0)
    top = s >= src - 1
    f, s = np.where(top, F32(0), f), np.where(top, src - 1, s)
    return s, np.minimum(s + 1, src - 1), f


def resize_linear_ref(img, out_hw, scale):
    """img [H, W, C] float -> fp64 [Hr, Wr, C]: cv2.resize(INTER_LINEAR) with cv2's coordinate rule and fp32 weights
    (horizontal pass, then vertical), the sums in fp64."""
    H, W = img.shape[:2]
    img = torch.as_tensor(img).double()
    ys0, ys1, fy = linear_coeffs(out_hw[0], H, 1.0 / scale)
    xs0, xs1, fx = linear_coeffs(out_hw[1], W, 1.0 / scale)
    fx = torch.from_numpy(fx.astype(np.float64))[None, :, None]
    fy = torch.from_numpy(fy.astype(np.float64))[:, None, None]
    rows = img[:, xs0] * (1 - fx) + img[:, xs1] * fx
    return rows[ys0] * (1 - fy) + rows[ys1] * fy


def linear_abs(img, out_hw, scale):
    """The same resize of |img|: the scale of its rounding errors."""
    return resize_linear_ref(np.abs(np.asarray(img, np.float64)), out_hw, scale)


def prep_ref(frames_u8, means, scale, out_hw, pad_hw):
    """frames [F, H, W, 3] uint8 -> fp64 [F, Hp, Wp, 3]: (pixel - mean) in fp32, resized unless the size is unchanged,
    zero padded to pad_hw."""
    Fn, H, W, _ = frames_u8.shape
    out = torch.zeros((Fn, pad_hw[0], pad_hw[1], 3), dtype=torch.float64)
    for f in range(Fn):
        im = frames_u8[f].astype(F32) - np.asarray(means, F32)
        v = torch.from_numpy(im).double() if tuple(out_hw) == (H, W) else resize_linear_ref(im, out_hw, scale)
        out[f, :out_hw[0], :out_hw[1]] = v
    return out


# ------------------------------------------------------------------ keypoint decode
def upsample2x_matrix(n):
    """[2n, n] fp64: the fixed bilinear ConvTranspose (kernel 4, stride 2, pad 1, filter [1, 3, 3, 1] / 4) in 1-D:
    out[o] = sum_i in[i] * f[o - 2i + 1]."""
    f = np.array([0.25, 0.75, 0.75, 0.25])
    U = np.zeros((2 * n, n))
    for o in range(2 * n):
        for i in range(n):
            k = o - 2 * i + 1
            if 0 <= k <= 3:
                U[o, i] = f[k]
    return torch.from_numpy(U)


def cubic_matrix(dst, src):
    """[dst, src] fp64: cv2.resize(INTER_CUBIC) along one axis, A = -0.75, replicated border, scale = 1 / (dst / src), the
    source coordinate and the four coefficients in fp32 as cv2 computes them."""
    A = F32(-0.75)
    scale = 1.0 / (float(dst) / src)
    f = ((np.arange(dst) + 0.5) * scale - 0.5).astype(F32)
    s = np.floor(f).astype(np.int64)
    x = f - s.astype(F32)
    x1 = x + F32(1)
    c0 = ((A * x1 - F32(5) * A) * x1 + F32(8) * A) * x1 - F32(4) * A
    c1 = ((A + F32(2)) * x - (A + F32(3))) * x * x + F32(1)
    y = F32(1) - x
    c2 = ((A + F32(2)) * y - (A + F32(3))) * y * y + F32(1)
    c3 = F32(1) - c0 - c1 - c2
    M = np.zeros((dst, src))
    for j, c in enumerate((c0, c1, c2, c3)):
        np.add.at(M, (np.arange(dst), np.clip(s - 1 + j, 0, src - 1)), c.astype(np.float64))
    return torch.from_numpy(M)


def decode_geometry(box, min_size):
    """One box (x1, y1, x2, y2) fp32 -> (rw, rh, wcorr, hcorr, offsets) as heatmaps_to_keypoints computes them."""
    b = np.asarray(box, F32)
    bw, bh = max(b[2] - b[0], F32(1)), max(b[3] - b[1], F32(1))
    rw, rh = int(np.ceil(bw)), int(np.ceil(bh))
    if min_size > 0:
        rw, rh = max(rw, min_size), max(rh, min_size)
    return rw, rh, F32(bw / F32(rw)), F32(bh / F32(rh)), b[0], b[1]


def keypoint_maps_ref(low, box, min_size=0):
    """low [K, 2S, 2S] (kps_score_lowres of one detection and frame) -> (heat [K, 4S, 4S] fp64, resized [K, rh, rw] fp64,
    |resized| scale, geometry): the 2x ConvTranspose, then cv2 INTER_CUBIC to (ceil(w), ceil(h)) as Ry @ M @ Rx^T."""
    low = low.double()
    n = low.shape[-1]
    U = upsample2x_matrix(n).to(low.device)
    heat = U @ low @ U.t()
    g = decode_geometry(box, min_size)
    Ry, Rx = cubic_matrix(g[1], 2 * n).to(low.device), cubic_matrix(g[0], 2 * n).to(low.device)
    return heat, Ry @ heat @ Rx.t(), Ry.abs() @ heat.abs() @ Rx.abs().t(), g


def keypoints_from_maps(res, g):
    """heatmaps_to_keypoints on fp64 resized maps [K, rh, rw]: first-index argmax, (x, y) in fp32 from the fp64 product
    (x_int + 0.5) * wcorr + offset, the logit and the softmax probability at the max -> [4, K] fp64, argmax [K]."""
    rw, rh, wc, hc, ox, oy = g
    K = res.shape[0]
    flat = res.reshape(K, -1)
    pos = flat.argmax(1)                        # torch returns the first maximal index
    mx = flat.max(1).values
    prob = 1.0 / torch.exp(flat - mx[:, None]).sum(1)
    xi, yi = (pos % rw).cpu().numpy(), (pos // rw).cpu().numpy()
    xy = np.zeros((4, K))
    xy[0] = ((xi + 0.5) * np.float64(wc) + np.float64(ox)).astype(F32)
    xy[1] = ((yi + 0.5) * np.float64(hc) + np.float64(oy)).astype(F32)
    xy[2], xy[3] = mx.cpu().numpy(), prob.cpu().numpy()
    return xy, pos


# ------------------------------------------------------------------ pooling, means, heads glue
def maxpool_ref(x, k, s, p):
    """[N, H, W, C] -> [N, Ho, Wo, C] (floor mode, -inf padding); the max is exact in any precision."""
    N, H, W, C = x.shape
    xp = F.pad(x.double(), (0, 0, p, p, p, p), value=float('-inf'))
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    out = None
    for dy in range(k):
        for dx in range(k):
            v = xp[:, dy:dy + s * (Ho - 1) + 1:s, dx:dx + s * (Wo - 1) + 1:s]
            out = v if out is None else torch.maximum(out, v)
    return out


def spatial_mean_seq(x):
    """[N, H, W, C] fp32 -> [N, C] fp32 by the kernel's documented order: per row a sequential sum over W, / W, the rows
    summed sequentially, / H (ReduceBackMean twice), every step one fp32 rounding."""
    x = x.float()
    N, H, W, C = x.shape
    acc = torch.zeros((N, C))
    for h in range(H):
        row = torch.zeros((N, C))
        for w in range(W):
            row = row + x[:, h, w]
        acc = acc + row / W
    return acc / H


def fold_tube_heads_ref(o, R, T, C):
    """o [R*T, ld] fp32 = per-frame [cls (C) | bbox (4C)] -> cls [R, C] = sequential fp32 sum over t / T, bbox [R, C*T*4]
    with channel c*4T + 4t + k."""
    o = o.float().view(R, T, -1)
    acc = o[:, 0, :C].clone()
    for t in range(1, T):
        acc = acc + o[:, t, :C]
    bbox = o[:, :, C:5 * C].reshape(R, T, C, 4).permute(0, 2, 1, 3).reshape(R, C * T * 4)
    return acc / T, bbox


def scale_rois_ref(boxes, ncols, im_scale, batch_idx=None, per_image=1):
    """[n, >= ncols] fp32 -> [n, ncols + 1] fp32: (image index, fp32(fp64(box) * im_scale))."""
    b = boxes[:, :ncols].double() * im_scale
    n = boxes.shape[0]
    idx = batch_idx.float() if batch_idx is not None else (torch.arange(n) // per_image).float()
    return torch.cat([idx[:, None].to(b.device), b.float()], 1)


# ================================================================== pins (CPU)
def _rand_rois(rng, R, T, nimg, W, H, out=False):
    x1, y1 = rng.uniform(-20 if out else 0, W - 2, R), rng.uniform(-20 if out else 0, H - 2, R)
    w, h = rng.uniform(0.3, W * 0.9, R), rng.uniform(0.3, H * 0.9, R)
    rois = np.zeros((R, 4 * T + 1), F32)
    rois[:, 0] = rng.integers(0, nimg, R)
    for t in range(T):
        j = rng.normal(0, 3, (R, 4)) * (t > 0)
        rois[:, 1 + 4 * t:5 + 4 * t] = np.stack([x1, y1, x1 + w, y1 + h], 1) + j
    return rois


@pytest.mark.parametrize('T,sampling', [(1, 2), (1, 0), (3, 2), (3, 0)])
def test_roi_align_matrix_vs_torchvision(T, sampling):
    """Forward S @ F and backward S^T @ G equal torchvision roi_align(aligned=False) and its autograd, two levels, two
    images, RoIs partly and wholly outside the map, widths below 1, and adaptive sampling."""
    from torchvision.ops import roi_align as tv
    g = torch.Generator().manual_seed(1)
    nimg, C, P = 2, 5, 7
    shapes = [(nimg * T, 20, 28), (nimg * T, 10, 14)]
    scales = [1 / 4., 1 / 8.]
    maps = [torch.randn(s + (C,), generator=g) for s in shapes]
    rng = np.random.default_rng(2)
    R = 40
    rois = _rand_rois(rng, R, T, nimg, 112, 80, out=True)
    rois[0, 1:5] = [200, 150, 260, 190]                          # wholly outside the map
    rois[1, 1:5] = [10, 10, 10.2, 10.1]                          # width and height below 1
    levels = rng.integers(2, 4, R).astype(np.int32)
    ref, A = roi_align_ref(maps, scales, rois, levels, P, sampling, T)
    G = torch.randn(ref.shape, generator=g, dtype=torch.float64)
    dF = A.unflat(A.S().t() @ G.reshape(-1, C))
    for t in range(T):
        for li in range(2):
            idx = np.where(levels == li + 2)[0]
            bt = torch.from_numpy(np.hstack([rois[idx, :1] * T + t, rois[idx, 1 + 4 * t:5 + 4 * t]]).astype(F32))
            fm = maps[li].permute(0, 3, 1, 2).contiguous().requires_grad_(True)
            out = tv(fm, bt, (P, P), scales[li], sampling, aligned=False)
            assert torch.allclose(out.double(), ref[idx, t].permute(0, 3, 1, 2), atol=1e-5, rtol=1e-5), (t, li)
            out.backward(G[idx, t].permute(0, 3, 1, 2).float())
            # the other frames' RoIs add to the same levels; compare the frame-t images of this level only
            imgs = [b * T + t for b in range(nimg)]
            got = dF[li][imgs]
            exp = fm.grad.permute(0, 2, 3, 1)[imgs].double()
            if T == 1:
                assert torch.allclose(got, exp, atol=1e-5, rtol=1e-5), (t, li)
            else:                                                # frame t's images receive only frame t's samples
                assert torch.allclose(got, exp, atol=1e-5, rtol=1e-5), (t, li)


def test_roi_align_matrix_marks_exact_geometry():
    """RoIs of width and height 7*2^j on a dyadic corner have exact fp32 geometry (no coordinate term); generic ones
    do not; samples land exactly on -1, 0, H-1 and H."""
    rois = np.array([[0, -4, -4, 52, 52], [0, 0.3, 0.7, 33.1, 40.9]], F32)     # scale 1/4: (-1, -1) to (13, 13)
    A = RoiAlignMatrix([(1, 12, 12)], [0.25], rois, None, 7, 2)
    assert np.all(A.ulp[:49] == 0) and np.all(A.ulp[49:] > 0)
    # bin 1 of row 0 samples at -1 + 2 * (0.5, 1.5) / 2 = -0.5, 0.5; bin 0 at -1 + (0.25, 0.75) * 2 = -0.5, 0.5
    S = A.S().to_dense()
    assert torch.isclose(S[0].sum(), torch.tensor(1.0, dtype=torch.float64))
    B = RoiAlignMatrix([(1, 12, 12)], [1.0], np.array([[0, -1, -1, 13, 13]], F32), None, 7, 1)
    assert np.all(B.ulp == 0)             # samples at -1 + 2*pw + 1: 0, 2, ..., 12 = H: inside the window, clamped


def test_resize_linear_vs_cv2():
    import cv2
    rng = np.random.default_rng(3)
    for (H, W), scale in (((45, 61), 1.6), ((45, 61), 0.53), ((36, 64), 1333 / 1280)):
        im = (rng.integers(0, 256, (H, W, 3)).astype(F32) - np.array([102.9801, 115.9465, 122.7717], F32))
        exp = cv2.resize(im, None, None, fx=scale, fy=scale, interpolation=cv2.INTER_LINEAR)
        got = resize_linear_ref(im, exp.shape[:2], scale)
        assert (got - torch.from_numpy(exp).double()).abs().max().item() <= 1e-4 * 255


def test_cubic_resize_vs_cv2():
    import cv2
    g = torch.Generator().manual_seed(4)
    m = torch.randn((56, 56), generator=g, dtype=torch.float64).float()
    for rw, rh in ((1, 1), (20, 37), (56, 56), (257, 300), (130, 90)):
        exp = cv2.resize(m.numpy(), (rw, rh), interpolation=cv2.INTER_CUBIC)
        got = cubic_matrix(rh, 56) @ m.double() @ cubic_matrix(rw, 56).t()
        assert (got - torch.from_numpy(exp).double()).abs().max().item() <= 1e-5 * m.abs().max().item()


def test_upsample_and_decode_vs_oracle():
    """The 2x ConvTranspose against oracle.keypoints.bilinear_upsample2x, and the decode against
    oracle.keypoints.heatmaps_to_keypoints (cv2), with min_size 0 and > 0."""
    from oracle import keypoints as ok
    g = torch.Generator().manual_seed(5)
    D, K = 4, 17
    low = F.avg_pool2d(torch.randn((D, K, 28, 28), generator=g), 3, 1, 1) * 3
    up = ok.bilinear_upsample2x(low)
    boxes = np.array([[10, 20, 60, 140], [5.5, 7.25, 300.2, 100.9], [0, 0, 0, 0], [100, 50, 103.5, 52]], F32)
    for min_size in (0, 8):
        exp = ok.heatmaps_to_keypoints(up.numpy(), boxes, K, min_size=min_size)
        for d in range(D):
            heat, res, _, geo = keypoint_maps_ref(low[d], boxes[d], min_size)
            assert (heat - up[d].double()).abs().max().item() <= 1e-6
            xy, _ = keypoints_from_maps(res, geo)
            assert np.allclose(xy[2], exp[d, 2], rtol=1e-5, atol=1e-5) and np.allclose(xy[3], exp[d, 3], rtol=1e-4)
            same = (xy[0].astype(F32) == exp[d, 0]) & (xy[1].astype(F32) == exp[d, 1])
            assert same.sum() >= K - 2
            for k in np.where(~same)[0]:                         # cv2's fp32 map picked a pixel that ties within fp32 noise
                rw, rh, wc, hc, ox, oy = geo
                xi = int(round((float(exp[d, 0, k]) - ox) / wc - 0.5)); yi = int(round((float(exp[d, 1, k]) - oy) / hc - 0.5))
                assert res[k, yi, xi].item() >= xy[2, k] - 1e-5 * res[k].abs().max().item()


def test_maxpool_ref_vs_torch():
    g = torch.Generator().manual_seed(6)
    x = torch.randn((3, 25, 41, 8), generator=g)
    for k, s, p in ((3, 2, 1), (1, 2, 0)):
        exp = F.max_pool2d(x.permute(0, 3, 1, 2), k, s, p).permute(0, 2, 3, 1)
        assert torch.equal(maxpool_ref(x, k, s, p).float(), exp)


def test_split_join_and_glue():
    g = torch.Generator().manual_seed(7)
    v = torch.randn((1000,), generator=g) * 100
    hi, lo = split_bf16(v)
    assert torch.equal(split_bf16(join(hi, lo))[0], hi) and torch.equal(split_bf16(join(hi, lo))[1], lo)
    assert ((join(hi, lo) - v).abs() <= 2.0 ** -16 * v.abs()).all()       # bf16 keeps 8 bits: 2^-8 twice
    th, tl = split_tf32(v)
    assert ((th.view(torch.int32) & 0x1FFF) == 0).all() and ((tl.view(torch.int32) & 0x1FFF) == 0).all()
    assert ((join(th, tl) - v).abs() <= 2.0 ** -22 * v.abs()).all()
    assert torch.equal(round_tf32(torch.tensor([1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11, -1 - 2.0 ** -11])),
                       torch.tensor([1.0, 1 + 2.0 ** -9, -1.0]))         # ties to even
    x = torch.randn((4, 3, 5, 8), generator=g)
    assert torch.allclose(spatial_mean_seq(x).double(), x.double().mean((1, 2)), atol=1e-6)
    o = torch.randn((6, 12), generator=g)
    cls, bbox = fold_tube_heads_ref(o, 2, 3, 2)
    assert torch.allclose(cls, o.view(2, 3, 12)[:, :, :2].mean(1), atol=1e-6)
    assert torch.equal(bbox[1, 1 * 12 + 2 * 4 + 3], o[1 * 3 + 2, 2 + 1 * 4 + 3])
    b = torch.tensor([[1.5, 2.0, 3.25, 4.0, 9.0]])
    assert torch.equal(scale_rois_ref(b, 4, 1.2), torch.tensor([[0, 1.8, 2.4, 3.9, 4.8]], dtype=torch.float64).float())
