"""Oracle: dense Farneback flow and flow-smoothed poses (TEST INFRASTRUCTURE ONLY).

Farneback: a numpy restatement of OpenCV 4.x's CPU ``calcOpticalFlowFarneback`` (modules/video/src/optflowgf.cpp)
with the OPTFLOW_FARNEBACK_GAUSSIAN window, stage by stage, with the filter taps built the way OpenCV builds them
(fp64, rounded to fp32) and the fp32 / fp64 arithmetic in OpenCV's order:
  bgr_to_gray            cvtColor BGR2GRAY, 15-bit fixed point
  gaussian_taps / gaussian_blur   GaussianBlur (reflect-101), the pyramid's pre-filter
  resize_linear          resize INTER_LINEAR (the exact 2x case is OpenCV's fast INTER_AREA)
  poly_exp               FarnebackPolyExp (n, sigma), replicate border
  update_matrices        FarnebackUpdateMatrices
  window_blur, solve_flow          FarnebackUpdateFlow_GaussianBlur (the window blur, the 2x2 solve)
  farneback              the pyramid driver
The build of OpenCV dispatches SIMD and IPP code, so cv2's last bits can differ from these by a few ulps per stage.

Smoothing: lib/core/tracking_engine.py:401-546 (_shift_using_flow, _shift_poses, _weighted_avg_poses,
_combine_boxes, _combine_shifted_poses) and :600-643 (_smooth_pose_video) with the flows supplied.
"""
import math

import numpy as np

F32 = np.float32


# ------------------------------------------------------------------------------------------------ gray conversion
def bgr_to_gray(bgr):
    """[.., 3] uint8 BGR -> uint8: (3735 B + 19235 G + 9798 R + 2^14) >> 15 (OpenCV 4.x's 15-bit coefficients)."""
    b = bgr[..., 0].astype(np.int32)
    g = bgr[..., 1].astype(np.int32)
    r = bgr[..., 2].astype(np.int32)
    return ((b * 3735 + g * 19235 + r * 9798 + (1 << 14)) >> 15).astype(np.uint8)


# ------------------------------------------------------------------------------------------------ pyramid
def gaussian_taps(ksize, sigma):
    """getGaussianKernel(ksize, sigma, CV_32F): fp32 taps; sigma <= 0 and ksize <= 7 take OpenCV's fixed tables."""
    fixed = {1: [1.0], 3: [0.25, 0.5, 0.25], 5: [0.0625, 0.25, 0.375, 0.25, 0.0625],
             7: [0.03125, 0.109375, 0.21875, 0.28125, 0.21875, 0.109375, 0.03125]}
    if sigma <= 0 and ksize in fixed:
        t = [F32(v) for v in fixed[ksize]]
    else:
        sx = sigma if sigma > 0 else ((ksize - 1) * 0.5 - 1) * 0.3 + 0.8
        s2 = -0.5 / (sx * sx)
        t = [F32(math.exp(s2 * (i - (ksize - 1) * 0.5) ** 2)) for i in range(ksize)]
    s = 0.0
    for v in t:
        s += float(v)
    s = 1.0 / s
    return np.array([F32(float(v) * s) for v in t], dtype=F32)


def _reflect101(i, n):
    i = np.abs(i)
    return np.where(i >= n, 2 * (n - 1) - i, i) if n > 1 else np.zeros_like(i)


def gaussian_blur(img, ksize, sigma):
    """GaussianBlur of an fp32 [H, W] image, ksize x ksize, reflect-101: a row pass (taps in ascending order) then
    a symmetric column pass."""
    k = gaussian_taps(ksize, sigma)
    r = ksize // 2
    H, W = img.shape
    cols = _reflect101(np.arange(-r, W + r), W)
    src = img[:, cols]
    row = src[:, 0:W] * k[0]
    for i in range(1, ksize):
        row = row + src[:, i:i + W] * k[i]
    rows = _reflect101(np.arange(-r, H + r), H)
    src = row[rows]
    out = src[r:r + H] * k[r]
    for i in range(1, r + 1):
        out = out + k[r + i] * (src[r + i:r + i + H] + src[r - i:r - i + H])
    return out.astype(F32)


def _linear_coeffs(dst, src):
    scale = 1.0 / (float(dst) / src)
    d = np.arange(dst, dtype=np.float64)
    f = ((d + 0.5) * scale - 0.5).astype(F32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(F32)).astype(F32)
    return s, f


def resize_linear(img, w, h):
    """resize(INTER_LINEAR) of fp32 [H, W] or [H, W, C] to (w, h).  Same size: a copy; exactly half: the fast
    2x2 average OpenCV switches to."""
    H, W = img.shape[:2]
    if (w, h) == (W, H):
        return img.copy()
    if W == 2 * w and H == 2 * h:
        a, b = img[0::2, 0::2], img[0::2, 1::2]
        c, d = img[1::2, 0::2], img[1::2, 1::2]
        return (((a + b) + (c + d)) * F32(0.25)).astype(F32)
    sx, fx = _linear_coeffs(w, W)
    lo = sx < 0
    fx[lo], sx[lo] = 0, 0
    hi = sx >= W - 1
    fx[hi], sx[hi] = 0, W - 1
    a1 = fx
    a0 = (F32(1) - fx).astype(F32)
    sx1 = np.minimum(sx + 1, W - 1)
    ex = img.ndim - 2
    a0x, a1x = a0.reshape((1, -1) + (1,) * ex), a1.reshape((1, -1) + (1,) * ex)
    hr = img[:, sx] * a0x + img[:, sx1] * a1x
    hr[:, hi] = img[:, sx[hi]]
    sy, fy = _linear_coeffs(h, H)
    b1 = fy
    b0 = (F32(1) - fy).astype(F32)
    y0 = np.clip(sy, 0, H - 1)
    y1 = np.clip(sy + 1, 0, H - 1)
    b0y, b1y = b0.reshape((-1, 1) + (1,) * ex), b1.reshape((-1, 1) + (1,) * ex)
    return (hr[y0] * b0y + hr[y1] * b1y).astype(F32)


# ------------------------------------------------------------------------------------------------ polynomial expansion
def poly_taps(n, sigma):
    """FarnebackPrepareGaussian: fp32 taps g, xg, xxg over -n..n and the fp64 entries ig11, ig03, ig33, ig55 of G^-1."""
    if sigma < np.finfo(np.float32).eps:
        sigma = n * 0.3
    x = np.arange(-n, n + 1)
    g = np.array([F32(math.exp(-(i * i) / (2 * sigma * sigma))) for i in x], dtype=F32)
    s = 0.0
    for v in g:
        s += float(v)
    s = 1.0 / s
    g = np.array([F32(float(v) * s) for v in g], dtype=F32)
    xg = np.array([F32(float(i) * float(v)) for i, v in zip(x, g)], dtype=F32)
    xxg = np.array([F32(float(i * i) * float(v)) for i, v in zip(x, g)], dtype=F32)
    G = np.zeros((6, 6))
    for yy in range(-n, n + 1):
        for xx in range(-n, n + 1):
            gg = float(g[yy + n]) * float(g[xx + n])
            G[0, 0] += gg
            G[1, 1] += gg * xx * xx
            G[3, 3] += gg * xx * xx * xx * xx
            G[5, 5] += gg * xx * xx * yy * yy
    G[2, 2] = G[0, 3] = G[0, 4] = G[3, 0] = G[4, 0] = G[1, 1]
    G[4, 4] = G[3, 3]
    G[3, 4] = G[4, 3] = G[5, 5]
    iG = np.linalg.inv(G)
    return g, xg, xxg, (iG[1, 1], iG[0, 3], iG[3, 3], iG[5, 5])


def poly_exp(img, n=7, sigma=1.5):
    """FarnebackPolyExp: fp32 [H, W] -> [H, W, 5] = (r_y, r_x, r_yy, r_xx, r_xy).  Column pass in fp32, row pass
    in fp64, replicate borders."""
    g, xg, xxg, (ig11, ig03, ig33, ig55) = poly_taps(n, sigma)
    g, xg, xxg = g[n:], xg[n:], xxg[n:]
    H, W = img.shape
    row0 = img * g[0]
    row1 = np.zeros_like(img)
    row2 = np.zeros_like(img)
    for k in range(1, n + 1):
        s0 = img[np.maximum(np.arange(H) - k, 0)]
        s1 = img[np.minimum(np.arange(H) + k, H - 1)]
        p = s0 + s1
        row0 = row0 + g[k] * p
        row1 = row1 + xg[k] * (s1 - s0)
        row2 = row2 + xxg[k] * p
    # the row pass accumulates in fp64, but OpenCV forms some products in fp32 first (float row x float tap)
    idx = np.clip(np.arange(-n, W + n), 0, W - 1)
    r0, r1, r2 = (r[:, idx] for r in (row0, row1, row2))
    c = slice(n, n + W)
    d = np.float64
    b1 = (r0[:, c] * g[0]).astype(d)
    b2 = np.zeros((H, W))
    b3 = (r1[:, c] * g[0]).astype(d)
    b4 = np.zeros((H, W))
    b5 = (r2[:, c] * g[0]).astype(d)
    b6 = np.zeros((H, W))
    for k in range(1, n + 1):
        p, m = slice(n + k, n + k + W), slice(n - k, n - k + W)
        tg = (r0[:, p] + r0[:, m]).astype(d)
        b1 = b1 + tg * float(g[k])
        b4 = b4 + tg * float(xxg[k])
        b2 = b2 + ((r0[:, p] - r0[:, m]) * xg[k]).astype(d)
        b3 = b3 + ((r1[:, p] + r1[:, m]) * g[k]).astype(d)
        b6 = b6 + ((r1[:, p] - r1[:, m]) * xg[k]).astype(d)
        b5 = b5 + ((r2[:, p] + r2[:, m]) * g[k]).astype(d)
    out = np.empty((H, W, 5), dtype=F32)
    out[..., 1] = b2 * ig11
    out[..., 0] = b3 * ig11
    out[..., 3] = b1 * ig03 + b4 * ig33
    out[..., 2] = b1 * ig03 + b5 * ig33
    out[..., 4] = b6 * ig55
    return out


# ------------------------------------------------------------------------------------------------ flow iterations
BORDER = np.array([0.14, 0.14, 0.4472, 0.4472, 0.4472], dtype=F32)


def _border_sides(n):
    """Per index, the attenuation of the low side and of the high side (1 outside the 5-pixel border)."""
    lo, hi = np.ones(n, dtype=F32), np.ones(n, dtype=F32)
    k = min(5, n)
    lo[:k] = BORDER[:k]
    hi[n - k:] = BORDER[:k][::-1]
    return lo, hi


def _border_scale(n):
    lo, hi = _border_sides(n)
    return lo * hi


def update_matrices(R0, R1, flow):
    """FarnebackUpdateMatrices: M [H, W, 5] = (G11, G12, G22, h1, h2) from R0, R1 sampled at x + flow."""
    H, W = flow.shape[:2]
    dx, dy = flow[..., 0], flow[..., 1]
    fx = np.arange(W, dtype=F32)[None, :] + dx
    fy = np.arange(H, dtype=F32)[:, None] + dy
    x1 = np.floor(fx).astype(np.int64)
    y1 = np.floor(fy).astype(np.int64)
    fx = fx - x1.astype(F32)
    fy = fy - y1.astype(F32)
    inside = (x1 >= 0) & (x1 < W - 1) & (y1 >= 0) & (y1 < H - 1)
    xa, ya = np.clip(x1, 0, W - 2), np.clip(y1, 0, H - 2)
    one = F32(1)
    a00, a01 = (one - fx) * (one - fy), fx * (one - fy)
    a10, a11 = (one - fx) * fy, fx * fy
    r = [a00 * R1[ya, xa, c] + a01 * R1[ya, xa + 1, c] + a10 * R1[ya + 1, xa, c] + a11 * R1[ya + 1, xa + 1, c]
         for c in range(5)]
    half, quarter = F32(0.5), F32(0.25)
    r2 = np.where(inside, r[0], F32(0))
    r3 = np.where(inside, r[1], F32(0))
    r4 = np.where(inside, (R0[..., 2] + r[2]) * half, R0[..., 2])
    r5 = np.where(inside, (R0[..., 3] + r[3]) * half, R0[..., 3])
    r6 = np.where(inside, (R0[..., 4] + r[4]) * quarter, R0[..., 4] * half)
    r2 = (R0[..., 0] - r2) * half
    r3 = (R0[..., 1] - r3) * half
    r2 = r2 + (r4 * dy + r6 * dx)
    r3 = r3 + (r6 * dy + r5 * dx)
    lo, hi = _border_sides(H)
    sc = (_border_scale(W)[None, :] * lo[:, None]) * hi[:, None]
    r2, r3, r4, r5, r6 = (v * sc for v in (r2, r3, r4, r5, r6))
    M = np.empty((H, W, 5), dtype=F32)
    M[..., 0] = r4 * r4 + r6 * r6
    M[..., 1] = (r4 + r5) * r6
    M[..., 2] = r5 * r5 + r6 * r6
    M[..., 3] = r4 * r2 + r6 * r3
    M[..., 4] = r6 * r2 + r5 * r3
    return M


def window_taps(winsize):
    """The fp32 half-kernel k[0..m] of FarnebackUpdateFlow_GaussianBlur (m = winsize // 2, sigma = 0.3 m)."""
    m = winsize // 2
    sigma = m * 0.3
    k = [F32(1.0)]
    s = 1.0
    for i in range(1, m + 1):
        k.append(F32(math.exp(-i * i / (2 * sigma * sigma))))
        s += float(k[i] * F32(2))
    s = 1.0 / s
    return np.array([F32(float(v) * s) for v in k], dtype=F32)


def window_blur(M, winsize):
    """The separable window blur of M: clamped columns (fp32 k0 * c + sum k_i (up + down)), then clamped rows."""
    k = window_taps(winsize)
    m = len(k) - 1
    H, W = M.shape[:2]
    v = M * k[0]
    for i in range(1, m + 1):
        v = v + (M[np.minimum(np.arange(H) + i, H - 1)] + M[np.maximum(np.arange(H) - i, 0)]) * k[i]
    h = v * k[0]
    for i in range(1, m + 1):
        h = h + k[i] * (v[:, np.maximum(np.arange(W) - i, 0)] + v[:, np.minimum(np.arange(W) + i, W - 1)])
    return h.astype(F32)


def solve_flow(S):
    """The regularised 2x2 solve of the blurred M, in fp64, rounded to fp32."""
    g11, g12, g22, h1, h2 = (S[..., c].astype(np.float64) for c in range(5))
    idet = 1.0 / (g11 * g22 - g12 * g12 + 1e-3)
    flow = np.empty(S.shape[:2] + (2,), dtype=F32)
    flow[..., 0] = (g11 * h2 - g12 * h1) * idet
    flow[..., 1] = (g22 * h1 - g12 * h2) * idet
    return flow


def level_sizes(H, W, pyr_scale=0.5, levels=10, min_size=32):
    """[(k, scale, w, h, blur ksize, blur sigma)] coarse to fine, as calcOpticalFlowFarneback lays out the pyramid."""
    scale, k = 1.0, 0
    while k < levels:
        scale *= pyr_scale
        if W * scale < min_size or H * scale < min_size:
            break
        k += 1
    out = []
    for lv in range(k, -1, -1):
        s = 1.0
        for _ in range(lv):
            s *= pyr_scale
        sigma = (1.0 / s - 1) * 0.5
        ks = max(int(np.rint(sigma * 5)) | 1, 3)
        out.append((lv, s, int(np.rint(W * s)), int(np.rint(H * s)), ks, sigma))
    return out


def farneback(gray0, gray1, pyr_scale=0.5, levels=10, winsize=None, iterations=10, poly_n=7, poly_sigma=1.5, trace=None):
    """calcOpticalFlowFarneback(gray0, gray1, None, ...) with OPTFLOW_FARNEBACK_GAUSSIAN: [H, W, 2] fp32.
    ``trace`` (a dict) receives the finest level's stages."""
    H, W = gray0.shape
    if winsize is None:
        winsize = min(H, W) // 5
    flow = None
    for lv, s, w, h, ks, sigma in level_sizes(H, W, pyr_scale, levels):
        if flow is None:
            flow = np.zeros((h, w, 2), dtype=F32)
        else:
            flow = resize_linear(flow, w, h) * F32(1.0 / pyr_scale)
        R = []
        for g in (gray0, gray1):
            I = resize_linear(gaussian_blur(g.astype(F32), ks, sigma), w, h)
            R.append(poly_exp(I, poly_n, poly_sigma))
        M = update_matrices(R[0], R[1], flow)
        for it in range(iterations):
            flow = solve_flow(window_blur(M, winsize))
            if it < iterations - 1:
                M = update_matrices(R[0], R[1], flow)
        if trace is not None and lv == 0:
            trace.update(R0=R[0], R1=R[1], flow=flow)
    return flow


# ------------------------------------------------------------------------------------------------ np.abs(flow).mean()
def pairwise_sum_f32(a):
    """numpy's float32 pairwise summation (8 accumulators in blocks of <= 128) of a 1-D float32 array."""
    a = np.ascontiguousarray(a, dtype=F32)
    n = len(a)
    if n < 8:
        r = F32(0)
        for v in a:
            r = F32(r + v)
        return r
    if n <= 128:
        r = a[:8].copy()
        i = 8
        while i < n - n % 8:
            r = r + a[i:i + 8]
            i += 8
        res = F32(F32(F32(r[0] + r[1]) + F32(r[2] + r[3])) + F32(F32(r[4] + r[5]) + F32(r[6] + r[7])))
        for v in a[i:]:
            res = F32(res + v)
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return F32(pairwise_sum_f32(a[:n2]) + pairwise_sum_f32(a[n2:]))


def flow_mean_abs(flow):
    """np.abs(flow).mean() of an fp32 flow, restated: fp32 pairwise sum over the flattened array, / size in fp32."""
    a = np.abs(np.ascontiguousarray(flow, dtype=F32)).ravel()
    return F32(F32(0) + pairwise_sum_f32(a)) / F32(a.size)


# ------------------------------------------------------------------------------------------------ smoothing
def shift_using_flow(poses, flow, boundary_th):
    """:401-428"""
    if flow is None:
        return []
    if np.abs(flow).mean() > boundary_th:
        return []
    res = []
    for pose in poses:
        res_pose = pose.copy()
        x = np.round(pose[0].copy())
        y = np.round(pose[1].copy())
        valid = (x >= 0) & (x < flow.shape[1]) & (y >= 0) & (y < flow.shape[0])
        x[~valid] = 0
        y[~valid] = 0
        dx = flow[y.astype('int'), x.astype('int'), 0]
        dy = flow[y.astype('int'), x.astype('int'), 1]
        dx[~valid] = 0
        dy[~valid] = 0
        res_pose[2, ~valid] = 0
        res_pose[0, :] += dx
        res_pose[1, :] += dy
        res.append(res_pose)
    return res


def shift_poses(pbt, delta, flows, boundary_th):
    """:431-451"""
    n = len(pbt)
    res = [([], [], [])] * n
    for f in range(n):
        t = f + delta
        if 0 <= t < n and len(pbt[f][0]) != 0:
            shifted = shift_using_flow(pbt[f][0], flows[f], boundary_th)
            if len(shifted) != 0:
                res[t] = (shifted, pbt[f][1], pbt[f][2])
    return res


def weighted_avg_poses(poses, shifts, K=17):
    """:454-462"""
    final = np.full((4, K), -np.inf, dtype=F32)
    for pose, shift in zip(poses, shifts):
        wt = pow(1.2, -abs(shift))
        if len(pose) > 0:
            good = pose[2, :] * wt > final[2, :]
            final[:, good] = pose[:, good]
            final[2, good] = final[2, good] * wt
    return final


def combine_boxes(boxes):
    """:465-479"""
    boxes = [b for b in boxes if len(b) > 0]
    assert len(boxes) > 0
    res = np.zeros_like(boxes[0])
    boxes = np.stack(boxes)
    score = np.max(boxes[:, -1])
    boxes = boxes[:, :-1]
    res[0::4] = np.min(boxes[:, 0::4], axis=0)
    res[1::4] = np.min(boxes[:, 1::4], axis=0)
    res[2::4] = np.max(boxes[:, 2::4], axis=0)
    res[3::4] = np.max(boxes[:, 3::4], axis=0)
    res[-1] = score
    return res


def combine_shifted(nframes, shifted, extend_tracks):
    """:482-546 without the debug hook."""
    out_p, out_b, out_t = [], [], []
    shifts = sorted(shifted.keys())
    for f in range(nframes):
        fp, fb, ft = [], [], []
        if extend_tracks:
            tracks = set()
            for s in shifts:
                tracks |= set(shifted[s][f][2])
            tracks = list(tracks)
        else:
            tracks = shifted[0][f][2]
        box_size = shifted[0][f][1].shape[-1]
        for t in tracks:
            po, bo = [], []
            for s in shifts:
                sp, sb, st = shifted[s][f]
                if t in st:
                    po.append(sp[st.index(t)])
                    bo.append(sb[st.index(t)])
                else:
                    po.append([])
                    bo.append([])
            fp.append(weighted_avg_poses(po, shifts))
            fb.append(combine_boxes(bo))
            ft.append(t)
        out_p.append(fp)
        out_b.append(np.stack(fb) if fb else np.zeros((0, box_size)))
        out_t.append(ft)
    return out_p, out_b, out_t


def smooth_pose_video(poses, boxes, tracks, flows, n_context, extend_tracks=True, boundary_th=6.0):
    """:600-643 for one video with the pair flows supplied (flows[i]: frame i -> i + 1, fp32 [H, W, 2] or None).
    Returns (poses, boxes, tracks) per frame."""
    import copy
    n = len(poses)
    if n_context > 0:
        fwd = list(flows) + [None]
        neg = [None] + [None if f is None else -f for f in flows]
    else:
        fwd = neg = []
    shifted = {0: copy.deepcopy(list(zip(poses, boxes, tracks)))}
    for i in range(1, n_context + 1):
        shifted[i] = shift_poses(shifted[i - 1], +1, fwd, boundary_th)
    for i in range(-n_context, 0)[::-1]:
        shifted[i] = shift_poses(shifted[i + 1], -1, neg, boundary_th)
    return combine_shifted(n, shifted, extend_tracks)
