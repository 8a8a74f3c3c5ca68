"""CPU: the references the training-step value tests (tests/test_gpu_train_step_ops.py) compare the non-GEMM kernels of
csrc/train_ops.cu with: the losses and their gradients, the pointwise backward joins, the FPN / stride-2 / slice-center
gradient plumbing, the sub-pixel deconv fix-up, the bias gradient and the momentum SGD update.  They are written from the
operators' documented semantics (Caffe2 SigmoidCrossEntropyLoss, SoftmaxWithLoss, AccuracyOp, MomentumSGDUpdate,
Detectron SmoothL1Loss, the spatial softmax through the fixed bilinear 2x ConvTranspose), share no code with the kernels,
and run as torch on either device.

Two kinds:
- exact emulations, for kernels whose result is one fixed fp32 operation order followed by one rounding: they apply that
  order in fp32, so the device must agree bit for bit;
- fp64 references with a bound per element, derived next to each one from the kernel's fp32 operation count (u = 2^-24,
  CUDA's expf within 2 ulp, logf / log1pf within 1, IEEE division; train_ops.cu is built without -fmad=false, so a bound
  allows for contraction).

Each reference is pinned here once on small shapes: the fp64 ones against torch autograd in fp64, the emulations against a
plain numpy restatement."""
import numpy as np
import torch
import torch.nn.functional as F

from test_dense_reference import U24, upsample2x_matrix

BF16_REL = 2.0 ** -8              # round to nearest bf16 (8 significant bits): |rounding| <= 2^-8 |v|
BF16_SUB = 2.0 ** -133            # bf16's smallest subnormal: the rounding of a stored value below bf16's normal range
TINY = 2.0 ** -126                # fp32's smallest normal: an expf that overflows / underflows loses at most this (times
#                                   the factor it is multiplied by); relative bounds stop holding below it


def f32(x):
    """A Python float as the fp32 the C ABI passes."""
    return float(np.float32(x))


def bf16_store_bound(acc, ref):
    """Bound of a value computed with error <= acc and stored in bf16: acc + the rounding of |ref| + acc."""
    return acc + BF16_REL * (ref.abs() + acc) + BF16_SUB


# ================================================================== exact emulations
def bwd_pointwise_ref(g1, g2=None, y=None, scale=None, second=False, scale2=None):
    """dt_bwd_pointwise(2): v = f32(g1) + f32(g2), zeroed unless y > 0 (Caffe2 ReluGradient: a NaN, -0 or +0 output masks);
    out = bf16(v * scale[c]) (or bf16(v)); out2 = bf16(v * scale2[c]) (or bf16(v)).  Returns out, or (out, out2)."""
    v = g1.float()
    if g2 is not None:
        v = v + g2.float()
    if y is not None:
        v = torch.where(y.float() > 0, v, torch.zeros_like(v))
    out = (v * scale.float() if scale is not None else v).bfloat16()
    if not second:
        return out
    return out, (v * scale2.float() if scale2 is not None else v).bfloat16()


def upsample_add_bwd_ref(fine, coarse=None):
    """dt_upsample_add_bwd: [..., 2Hc, 2Wc, C] -> bf16(((((0 + c00) + c01) + c10) + c11) + coarse) in fp32, children
    (dy, dx) in row-major order."""
    f = fine.float()
    v = torch.zeros_like(f[..., 0::2, 0::2, :])
    for dy in (0, 1):
        for dx in (0, 1):
            v = v + f[..., dy::2, dx::2, :]
    if coarse is not None:
        v = v + coarse.float()
    return v.bfloat16()


def grad_join_ref(acc, g=None):
    """dt_grad_join_f32: bf16(acc + f32(g))."""
    return (acc + g.float() if g is not None else acc).bfloat16()


def scatter_stride2_ref(src, H, W):
    """dt_scatter_stride2: src [..., ceil(H/2), ceil(W/2), C] on the even positions of a zero [..., H, W, C] map."""
    out = torch.zeros(tuple(src.shape[:-3]) + (H, W, src.shape[-1]), dtype=src.dtype, device=src.device)
    out[..., 0::2, 0::2, :] = src
    return out


def embed_frame_ref(src, T, c):
    """dt_embed_frame: src [B, ...] as frame c of [B, T, ...], every other frame zero."""
    out = torch.zeros((src.shape[0], T) + tuple(src.shape[1:]), dtype=src.dtype, device=src.device)
    out[:, c] = src
    return out


def subpixel_live(K, ldc):
    """[9, ldc] bool: tap (dy, dx) of the 3 x 3 footprint is live for output channel co = sub * K + k (sub = 2 py + px)
    iff the 4 x 4 ConvTranspose (stride 2, pad 1) tap it stands for, (py + 1 - 2 dy, px + 1 - 2 dx), lies inside the
    kernel; channels >= 4K are padding."""
    live = torch.zeros((9, ldc), dtype=torch.bool)
    for sub in range(4):
        py, px = sub >> 1, sub & 1
        for tap in range(9):
            dy, dx = tap // 3 - 1, tap % 3 - 1
            if 0 <= py + 1 - 2 * dy <= 3 and 0 <= px + 1 - 2 * dx <= 3:
                live[tap, sub * K:(sub + 1) * K] = True
    return live


def subpixel_fix_ref(gW, gb, K):
    """dt_subpixel_grad_fix: dead taps of gW [9, ldc, Cin] zeroed; the four sub-pixel copies of each bias gradient replaced
    by their sum ((b0 + b1) + b2) + b3 in fp32; bias channels [4K, ldc) zeroed.  Returns (gW, gb)."""
    ldc = gW.shape[1]
    live = subpixel_live(K, ldc).to(gW.device)
    w = torch.where(live[:, :, None], gW, torch.zeros_like(gW))
    if gb is None:
        return w, None
    s = ((gb[0:K] + gb[K:2 * K]) + gb[2 * K:3 * K]) + gb[3 * K:4 * K]
    b = torch.zeros_like(gb)
    b[:4 * K] = s.repeat(4)
    return w, b


# ================================================================== fp64 references with bounds
def rpn_loss_ref(out, labels, tgt, iw, ow, A, s_cls, s_box, beta):
    """FPN RPN losses of one level (SigmoidCrossEntropyLoss(normalize=0) + SmoothL1Loss(beta)), fp64:
    out [rows, >= 5A] = [A logits | 4A deltas], labels [rows, A] (-1 ignore).  Returns (grad cls [rows, A] (zero where
    ignored), grad box [rows, 4A], cls loss, box loss)."""
    out = out.double()
    x = out[:, :A]
    t = labels.double()
    valid = labels >= 0
    lc = s_cls * (torch.clamp(x, min=0) - x * t + torch.log1p(torch.exp(-x.abs())))
    gc = s_cls * (torch.sigmoid(x) - t)
    d = iw.double() * (out[:, A:5 * A] - tgt.double())
    ad = d.abs()
    lb = s_box * ow.double() * torch.where(ad < beta, 0.5 * d * d / beta, ad - 0.5 * beta)
    gb = s_box * ow.double() * iw.double() * torch.where(ad < beta, d / beta, torch.sign(d))
    return (torch.where(valid, gc, torch.zeros_like(gc)), gb, float(torch.where(valid, lc, torch.zeros_like(lc)).sum()),
            float(lb.sum()))


def rpn_loss_terms(out, labels, tgt, iw, ow, A, s_cls, s_box, beta):
    """The per-element loss terms [rows, 5A] of rpn_loss_ref (0 where ignored), for the summation bound."""
    o = out.double()
    x, t = o[:, :A], labels.double()
    lc = s_cls * (torch.clamp(x, min=0) - x * t + torch.log1p(torch.exp(-x.abs())))
    d = iw.double() * (o[:, A:5 * A] - tgt.double())
    ad = d.abs()
    lb = s_box * ow.double() * torch.where(ad < beta, 0.5 * d * d / beta, ad - 0.5 * beta)
    return torch.cat([torch.where(labels >= 0, lc, torch.zeros_like(lc)), lb], 1)


def rpn_grad_bound(out, labels, tgt, iw, ow, A, s_cls, s_box, beta):
    """Per-element bound [rows, 5A] of dt_rpn_loss_grad's bf16 gradient against rpn_loss_ref (beta: the fp32 value).
    cls, s_cls * (1 / (1 + expf(-x)) - t): expf 2 ulp (4u, scaled by e / (1 + e) <= 1), the add and the division u each:
    sigma to 6u sigma; the subtraction and the product u |.| each; plus s_cls * TINY for expf's overflow (x < -88.7, sigma
    flushed to 0) and underflow.  box, s_box * w_out * w_in * (|d| < beta ? d / beta : sign d): d = w_in * (o - t) to 2u,
    d / beta and three products u each: 6u of the magnitude; where |d| lies within d's 2u of beta the two branches differ
    by <= 2u |d| / beta, so the bound is 8u * s_box |w_out w_in| min(|d| / beta, 1) on both sides of the seam."""
    o = out.double()
    x, t = o[:, :A], labels.double()
    sig = torch.sigmoid(x)
    acc_c = s_cls * (6 * U24 * sig + 2 * U24 * (sig - t).abs() + TINY)
    acc_c = torch.where(labels >= 0, acc_c, torch.zeros_like(acc_c))
    d = iw.double() * (o[:, A:5 * A] - tgt.double())
    acc_b = 8 * U24 * s_box * (ow.double() * iw.double()).abs() * torch.clamp(d.abs() / beta, max=1.0)
    gc, gb, _, _ = rpn_loss_ref(out, labels, tgt, iw, ow, A, s_cls, s_box, beta)
    return bf16_store_bound(torch.cat([acc_c, acc_b], 1), torch.cat([gc, gb], 1))


def rpn_loss_bound(terms, start, rows, ld_g, num_sms):
    """Bound of the loss sum of one dt_rpn_loss_grad launch accumulated onto `start`.  Each term: cls through expf, log1pf
    (1 ulp) and 4 operations, box through 7 operations on d (2u): <= 10u |term| (+ s * TINY in the underflow range, inside
    the 10u of the largest term for these scales).  The sum: each thread adds its grid-stride terms in order, a 5-level warp
    shuffle tree, then one atomicAdd per warp in any order onto start: depth = per-thread terms + 5 + warps, each level one
    rounding of a partial sum <= |start| + sum |terms| (a standard bound for any summation order of that depth)."""
    total = rows * ld_g
    grid = min(-(-total // 256), num_sms * 16)
    per = -(-total // (grid * 256))
    depth = per + 5 + grid * 8
    a = float(terms.abs().sum())
    return 10 * U24 * a + depth * U24 * (abs(start) + a)


def frcnn_loss_ref(out, labels, tgt, iw, ow, C, N, s_cls, s_box):
    """Fast R-CNN head losses (Caffe2 SoftmaxWithLoss over C classes + Detectron SmoothL1Loss with beta 1, both normalised
    by N = totals[0]), fp64, on out [rows, >= 5C] = [C logits | 4C deltas], labels [rows] (-1: padding row).  Returns
    (grad [rows, 5C], cls loss per row, box loss per row, hit per row: Caffe2 AccuracyOp's top-1 with the FIRST maximum
    winning a tie, on the fp32 logits), everything zero on padding rows and when N == 0."""
    o = out.double()
    x = o[:, :C]
    live = (labels >= 0) & (N > 0)
    lbl = labels.clamp_min(0).long()
    k_c, k_b = (s_cls / N, s_box / N) if N > 0 else (0.0, 0.0)
    lsm = torch.log_softmax(x, 1)
    gc = (lsm.exp() - F.one_hot(lbl, C).double()) * k_c
    d = iw.double() * (o[:, C:5 * C] - tgt.double())
    ad = d.abs()
    gb = ow.double() * iw.double() * torch.where(ad < 1, d, torch.sign(d)) * k_b
    lc = -lsm.gather(1, lbl[:, None])[:, 0] * k_c
    lb = (ow.double() * torch.where(ad < 1, 0.5 * d * d, ad - 0.5)).sum(1) * k_b
    idx = torch.arange(C, device=x.device)
    first = torch.where(x == x.max(1, keepdim=True).values, idx, C).min(1).values
    z = lambda v: torch.where(live.view((-1,) + (1,) * (v.dim() - 1)), v, torch.zeros_like(v))
    return z(torch.cat([gc, gb], 1)), z(lc), z(lb), (first == lbl) & live


def frcnn_bounds(out, labels, tgt, iw, ow, C, N, s_cls, s_box):
    """(grad bound [rows, 5C], cls loss term bound [rows], box loss term bound [rows]) of dt_frcnn_loss_grad against
    frcnn_loss_ref.  Per row the kernel takes m = max x (exact), se = sum_j expf(x_j - m) (C expf of 4u, the arguments'
    subtraction u |x_j - m|, C - 1 additions), lse = logf(se) (1 ulp): lse off by E = sum_j p_j u |x_j - m| + (C + 3)u +
    2u |lse|; p_i = expf(x_i - m - lse) then carries eps_i = u |x_i - m| + u |x_i - m - lse| + E + 4u relative, and
    (p_i - [i == label]) * s / N three more roundings of its magnitude, + s / N * TINY where expf underflows.  The box
    gradient as rpn_grad_bound with beta 1 and 4 products.  Loss terms: -(x_l - m - lse) * s / N to its argument's error
    + 2u; the box loss of a row adds 4C terms of <= 10u each in order (4C roundings of the running sum)."""
    o = out.double()
    x = o[:, :C]
    live = ((labels >= 0) & (N > 0)).double()
    k_c, k_b = (s_cls / N, s_box / N) if N > 0 else (0.0, 0.0)
    m = x.max(1, keepdim=True).values
    dm = x - m
    lse = torch.logsumexp(dm, 1, keepdim=True)
    p = torch.exp(dm - lse)
    E = (p * U24 * dm.abs()).sum(1, keepdim=True) + (C + 3) * U24 + 2 * U24 * lse.abs()
    eps = U24 * dm.abs() + U24 * (dm - lse).abs() + E + 4 * U24
    lbl = labels.clamp_min(0).long()
    t = F.one_hot(lbl, C).double()
    acc_c = k_c * (p * eps + 3 * U24 * (p - t).abs() + TINY)
    d = iw.double() * (o[:, C:5 * C] - tgt.double())
    acc_b = 8 * U24 * k_b * (ow.double() * iw.double()).abs() * torch.clamp(d.abs(), max=1.0)
    ref, lc, lb, _ = frcnn_loss_ref(out, labels, tgt, iw, ow, C, N, s_cls, s_box)
    g = bf16_store_bound(torch.cat([acc_c, acc_b], 1) * live[:, None], ref)
    arg = (dm - lse).gather(1, lbl[:, None])[:, 0]
    b_lc = (k_c * (U24 * dm.gather(1, lbl[:, None])[:, 0].abs() + U24 * arg.abs() + E[:, 0]) + 2 * U24 * lc.abs()) * live
    ad = d.abs()
    lb_terms = (ow.double() * torch.where(ad < 1, 0.5 * d * d, ad - 0.5)).abs() * k_b
    b_lb = (10 * U24 + 4 * C * U24) * lb_terms.sum(1) * live
    return g, b_lc, b_lb


def unpack_low(low, K):
    """kps_score_lowres in the sub-pixel packed layout [D, S, S, >= 4K] (channel (2 py + px) K + k at (y, x) holds map
    pixel (2y + py, 2x + px) of joint k) -> [D, K, 2S, 2S]."""
    D, S = low.shape[0], low.shape[1]
    x = low[..., :4 * K].reshape(D, S, S, 2, 2, K)
    return x.permute(0, 5, 1, 3, 2, 4).reshape(D, K, 2 * S, 2 * S)


def pack_low(m, ld):
    """unpack_low's inverse, zero in channels [4K, ld)."""
    D, K, S2 = m.shape[0], m.shape[1], m.shape[2]
    S = S2 // 2
    out = torch.zeros((D, S, S, ld), dtype=m.dtype, device=m.device)
    out[..., :4 * K] = m.reshape(D, K, S, 2, S, 2).permute(0, 2, 4, 3, 5, 1).reshape(D, S, S, 4 * K)
    return out


def kps_loss_ref(low, K, loc, w, tw, scale, ld_g):
    """Keypoint head loss (the spatial SoftmaxWithLoss over the 4S x 4S map after the fixed bilinear 2x ConvTranspose,
    weighted by w / sum w), fp64: U = R L R^T per (RoI, joint) with R = upsample2x_matrix(2S); dL = R^T (p - e_t) R *
    w * scale / tw, packed like `low` into [D, S, S, ld_g].  Returns (grad, loss per (RoI, joint), a dict of the
    intermediates kps_bounds needs)."""
    D, S = low.shape[0], low.shape[1]
    M = 4 * S
    R = upsample2x_matrix(2 * S).to(low.device)
    Lm = unpack_low(low.double(), K)
    U = (R @ Lm @ R.t()).reshape(D, K, M * M)
    lsm = torch.log_softmax(U, -1)
    p = lsm.exp()
    live = (w > 0) & (tw > 0)
    gs = torch.where(live, w.double() * scale / max(tw, 1e-300), torch.zeros_like(w.double()))
    e = torch.zeros_like(p)
    e.scatter_(2, loc.long()[..., None], 1.0)
    dU = (p - e) * gs[..., None]
    dL = R.t() @ dU.view(D, K, M, M) @ R
    loss = -lsm.gather(2, loc.long()[..., None])[..., 0] * gs
    return pack_low(dL, ld_g), loss, dict(R=R, Lm=Lm, U=U, lsm=lsm, p=p, e=e, gs=gs, dU=dU)


def kps_bounds(ref, it, ld_g):
    """(grad bound [D, S, S, ld_g], loss term bound [D, K]) of dt_kps_loss_grad against kps_loss_ref, element by element.
    U: <= 4 terms L * f * f (two roundings each, or one inside an FMA) added from 0 (<= 3 roundings): eU = 5u (R |L| R^T).
    The sum s = sum_j expf(U_j - mx) runs over 4S^2 / 256 <= 13 terms per thread, a 5-level shuffle and 8 warp partials:
    26 roundings of a positive sum, each term 4u (expf) + u |U_j - mx| + eU_j; lse = logf(s) adds 1 ulp (2u |lse|); mx
    cancels between s and p.  p_i = expf(U_i - mx - lse): eps_i = eU_i + u |U_i - mx| + u |U_i - mx - lse| + err(lse) + 4u.
    dU_i = (p_i - [i == t]) * gs, gs = w * scale / tw in fp32 (2 roundings): gs (p_i eps_i + 4u |p_i - t_i| + TINY).
    dL: 16 terms dU * f * f (2 roundings each) added from 0 (15): 17u of R^T |dU| R, plus R^T err(dU) R; then bf16."""
    R, U, p, e, gs, dU = it['R'], it['U'], it['p'], it['e'], it['gs'], it['dU']
    D, K = gs.shape
    M = R.shape[0]
    eU = 5 * U24 * (R @ it['Lm'].abs() @ R.t()).reshape(D, K, M * M)
    dm = U - U.max(-1, keepdim=True).values
    lse = torch.logsumexp(dm, -1, keepdim=True)
    err_lse = (p * (eU + U24 * dm.abs())).sum(-1, keepdim=True) + 30 * U24 + 2 * U24 * lse.abs()
    eps = eU + U24 * dm.abs() + U24 * (dm - lse).abs() + err_lse + 4 * U24
    e_dU = gs[..., None] * (p * eps + 4 * U24 * (p - e).abs() + TINY)
    acc = R.t() @ e_dU.view(D, K, M, M) @ R + 17 * U24 * (R.t() @ dU.abs().view(D, K, M, M) @ R)
    g = bf16_store_bound(pack_low(acc, ld_g), ref)
    t_arg = (dm - lse)
    tsel = lambda v: (v * e).sum(-1)
    b_loss = gs * (tsel(eU) + U24 * tsel(dm.abs()) + U24 * tsel(t_arg.abs()) + err_lse[..., 0]) + 3 * U24 * (gs * tsel(t_arg.abs()))
    return g, b_loss


def sgd_ref(w, g, m, lr, momentum, wd, grad_scale, lr_mult=1.0, wd_mult=1.0):
    """Caffe2 MomentumSGDUpdate (non-Nesterov) after the WeightedSum weight decay, fp64, with the item's lr / wd multipliers
    applied in fp32 as the kernel does: adj = lr_i (gs g + wd_i w) + mu m; m' = adj; w' = w - adj.  Returns (w', m', bound w',
    bound m').  Bound: a = gs g and b = wd_i w one rounding each, a + b one, lr_i * that one (3u lr_i (|a| + |b|) in all),
    q = mu m one, adj one more of |adj|; w' one more of |w'|.  Contraction only removes roundings; (1 + 2^-20) covers the
    second-order terms and fp64's own."""
    lr_i, wd_i = f32(f32(lr) * f32(lr_mult)), f32(f32(wd) * f32(wd_mult))
    mu, gs = f32(momentum), f32(grad_scale)
    w, g, m = w.double(), g.double(), m.double()
    a, b, q = gs * g, wd_i * w, mu * m
    adj = lr_i * (a + b) + q
    nw = w - adj
    bm = U24 * (3 * lr_i * (a.abs() + b.abs()) + q.abs() + adj.abs()) * (1 + 2.0 ** -20)
    return nw, adj, bm + U24 * nw.abs() * (1 + 2.0 ** -20), bm


def bias_grad_bound(g, db0, rows, num_sms):
    """Bound of dt_bias_grad (db += sum over rows of g[row, c]) per channel: gx = min(max(rows / 128, 1), 8 SMs) row blocks,
    8 row lanes each adding ceil(ceil(rows / gx) / 8) values in order, 8 lane partials, one atomicAdd per block in any order:
    depth = that + 8 + gx roundings of a partial <= |db0| + sum |g|."""
    gx = min(max(rows // 128, 1), num_sms * 8)
    per = -(-rows // gx)
    depth = -(-per // 8) + 8 + gx
    return depth * U24 * (db0.double().abs() + g.double().abs().sum(0))


# ================================================================== pins
def _bf16_np(x):
    """fp32 -> bf16 (as fp32) by round to nearest even on the bit pattern (finite values)."""
    u = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return r.astype(np.uint32).view(np.float32)


def _edges_bf16(g, n):
    """n bf16 values: random, +-0, the smallest subnormal, and pairs whose fp32 sum is a bf16 rounding tie."""
    v = torch.randn(n, generator=g).bfloat16()
    v[:6] = torch.tensor([0.0, -0.0, 2.0 ** -133, -2.0 ** -133, 1 + 2 ** -7, 2 ** -8]).bfloat16()
    return v


def test_bwd_pointwise_ref_vs_numpy_restatement():
    g = torch.Generator().manual_seed(1)
    C = 16
    g1, g2, y = (_edges_bf16(g, 4 * C).view(4, C) for _ in range(3))
    g2[0, :6] = -g1[0, :6]                                       # exact cancellation
    y[1, :4] = torch.tensor([0.0, -0.0, 2.0 ** -133, float('nan')]).bfloat16()
    sc, sc2 = torch.rand(C, generator=g) + 0.5, torch.rand(C, generator=g) + 0.5
    sc[:2] = 1.0
    out, out2 = bwd_pointwise_ref(g1, g2, y, sc, second=True, scale2=sc2)
    a, b, yy = g1.float().numpy(), g2.float().numpy(), y.float().numpy()
    for r in range(4):
        for c in range(C):
            v = np.float32(a[r, c]) + np.float32(b[r, c])
            v = v if yy[r, c] > 0 else np.float32(0)
            assert out[r, c].float().item() == _bf16_np(np.float32(v * np.float32(sc[c].item()))), (r, c)
            assert out2[r, c].float().item() == _bf16_np(np.float32(v * np.float32(sc2[c].item()))), (r, c)
    assert torch.equal(bwd_pointwise_ref(g1), g1)
    o1, o2 = bwd_pointwise_ref(g1, None, y, sc, second=True)
    assert torch.equal(o2, torch.where(y.float() > 0, g1.float(), torch.zeros(1)).bfloat16())
    # the tie: 1 + 2^-7 + 2^-8 rounds to the even neighbour 1 + 2^-6 in bf16
    assert float(bwd_pointwise_ref(torch.tensor([1 + 2 ** -7]).bfloat16(), torch.tensor([2 ** -8]).bfloat16())) == 1 + 2 ** -6


def test_upsample_add_and_joins_vs_numpy_restatement():
    g = torch.Generator().manual_seed(2)
    fine = torch.randn((2, 4, 6, 8), generator=g).bfloat16()
    coarse = torch.randn((2, 2, 3, 8), generator=g).bfloat16()
    fine[0, 0:2, 0:2, 0] = torch.tensor([[2.0 ** 24, 2.0 ** 16], [1.0, 1.0]]).bfloat16()     # order-sensitive magnitudes
    coarse[0, 0, 0, 0] = 0
    got = upsample_add_bwd_ref(fine, coarse)
    f, c = fine.float().numpy(), coarse.float().numpy()
    for i in np.ndindex(c.shape):
        n, h, w, ch = i
        v = np.float32(0)
        for dy in (0, 1):
            for dx in (0, 1):
                v = np.float32(v + f[n, 2 * h + dy, 2 * w + dx, ch])
        v = np.float32(v + c[i])
        assert got[i].float().item() == _bf16_np(v), i
    assert got[0, 0, 0, 0].float().item() == 2.0 ** 24          # the sum order's tie; (c10 + c11) first gives 2^24 + 2^17
    acc = torch.randn((4, 8), generator=g)
    gb = torch.randn((4, 8), generator=g).bfloat16()
    assert np.array_equal(grad_join_ref(acc, gb).float().numpy(), _bf16_np(acc.numpy() + gb.float().numpy()))
    src = torch.randn((2, 1, 3, 4, 8), generator=g)
    sc = scatter_stride2_ref(src, 5, 7)
    for h in range(5):
        for w in range(7):
            exp = src[:, :, h // 2, w // 2] if (h % 2 == 0 and w % 2 == 0) else torch.zeros_like(src[:, :, 0, 0])
            assert torch.equal(sc[:, :, h, w], exp)
    e = embed_frame_ref(src[:, 0], 3, 1)
    assert torch.equal(e[:, 1], src[:, 0]) and not e[:, 0].any() and not e[:, 2].any()


def test_subpixel_live_taps_are_the_deconv_taps():
    """A ConvTranspose k4 s2 p1 equals four 3 x 3 convs (one per output sub-pixel) whose live taps are subpixel_live's:
    the fix-up's mask is the decomposition the trainer's kps_score_lowres filter uses."""
    g = torch.Generator().manual_seed(3)
    K, ldc = 1, 8
    x = torch.randn((1, 1, 6, 7), generator=g, dtype=torch.float64)
    wt = torch.randn((1, 1, 4, 4), generator=g, dtype=torch.float64)
    ref = F.conv_transpose2d(x, wt, stride=2, padding=1)               # [1, 1, 12, 14]
    live = subpixel_live(K, ldc)
    for sub in range(4):
        py, px = sub >> 1, sub & 1
        w3 = torch.zeros((1, 1, 3, 3), dtype=torch.float64)
        for tap in range(9):
            dy, dx = tap // 3 - 1, tap % 3 - 1
            if live[tap, sub]:
                w3[0, 0, dy + 1, dx + 1] = wt[0, 0, py + 1 - 2 * dy, px + 1 - 2 * dx]
        assert torch.allclose(F.conv2d(x, w3, padding=1), ref[:, :, py::2, px::2], rtol=0, atol=1e-12), sub
    assert int(live[:, :4 * K].sum()) == 16 and not live[:, 4 * K:].any()
    gW = torch.randn((9, ldc, 5), generator=g)
    gb = torch.randn(ldc, generator=g)
    w, b = subpixel_fix_ref(gW, gb, K)
    assert torch.equal(w[~live], torch.zeros_like(w[~live])) and torch.equal(w[live], gW[live])
    s = np.float32(np.float32(np.float32(gb[0].item()) + np.float32(gb[1].item())) + np.float32(gb[2].item())) + np.float32(gb[3].item())
    assert (b[:4] == float(np.float32(s))).all() and not b[4:].any()


def test_rpn_loss_ref_vs_autograd():
    g = torch.Generator().manual_seed(4)
    rows, A, beta = 200, 3, f32(1.0 / 9.0)
    out = torch.randn((rows, 16), generator=g, dtype=torch.float64) * 3
    out[:6, 0] = torch.tensor([0.0, 1e-3, -1e-3, 17.0, -17.0, 90.0], dtype=torch.float64)
    labels = torch.randint(-1, 2, (rows, A), generator=g, dtype=torch.int32)
    tgt = out[:, A:5 * A] + (torch.rand((rows, 4 * A), generator=g, dtype=torch.float64) - 0.5) * 0.5
    iw = (torch.rand((rows, 4 * A), generator=g) > 0.3).double()
    ow = (torch.rand((rows, 4 * A), generator=g) > 0.2).double() / 256
    s_cls, s_box = 1.0 / 512, 0.5
    gc, gb, lc, lb = rpn_loss_ref(out, labels, tgt, iw, ow, A, s_cls, s_box, beta)
    o = out.clone().requires_grad_(True)
    valid = (labels >= 0).double()
    l_c = (F.binary_cross_entropy_with_logits(o[:, :A], labels.double().clamp_min(0), reduction='none') * valid).sum() * s_cls
    d = iw * (o[:, A:5 * A] - tgt)
    ad = d.abs()
    l_b = (ow * torch.where(ad < beta, 0.5 * d * d / beta, ad - 0.5 * beta)).sum() * s_box
    (l_c + l_b).backward()
    l_c, l_b = float(l_c.detach()), float(l_b.detach())
    assert abs(lc - l_c) <= 1e-12 * abs(l_c) and abs(lb - l_b) <= 1e-12 * abs(l_b)
    assert torch.allclose(torch.cat([gc, gb], 1), o.grad[:, :5 * A], rtol=1e-12, atol=1e-300)
    assert torch.allclose(rpn_loss_terms(out, labels, tgt, iw, ow, A, s_cls, s_box, beta).sum(), torch.tensor(lc + lb, dtype=torch.float64))


def test_frcnn_loss_ref_vs_autograd():
    g = torch.Generator().manual_seed(5)
    rows, C, N = 100, 3, 70.0
    out = torch.randn((rows, 16), generator=g) * 3
    out[0, :C] = torch.tensor([2.0, 2.0, 1.0])                         # tie: the first maximum wins
    out[1, :C] = torch.tensor([1.0, 4.0, 4.0])
    labels = torch.randint(0, C, (rows,), generator=g, dtype=torch.int32)
    labels[0], labels[1], labels[70:] = 1, 1, -1
    tgt = torch.randn((rows, 4 * C), generator=g) * 2
    iw = (torch.rand((rows, 4 * C), generator=g) > 0.5).float()
    ow = iw.clone()
    grad, lc, lb, hit = frcnn_loss_ref(out, labels, tgt, iw, ow, C, N, 0.5, 0.25)
    o = out.double().clone().requires_grad_(True)
    live = labels >= 0
    l_c = F.cross_entropy(o[live][:, :C], labels[live].long(), reduction='sum') * 0.5 / N
    d = iw.double() * (o[:, C:5 * C] - tgt.double())
    ad = d.abs()
    l_b = (ow.double() * torch.where(ad < 1, 0.5 * d * d, ad - 0.5))[live].sum() * 0.25 / N
    (l_c + l_b).backward()
    l_c, l_b = float(l_c.detach()), float(l_b.detach())
    assert torch.allclose(grad, o.grad[:, :5 * C], rtol=1e-12, atol=1e-300)
    assert abs(float(lc.sum()) - l_c) <= 1e-12 * l_c and abs(float(lb.sum()) - l_b) <= 1e-12 * l_b
    assert not bool(hit[0]) and bool(hit[1])                          # ties resolve to the first maximum: 0, then 1
    assert int(hit[2:70].sum()) == int((out[2:70, :C].argmax(1) == labels[2:70]).sum())
    assert not frcnn_loss_ref(out, labels, tgt, iw, ow, C, 0.0, 0.5, 0.25)[0].any()


def test_kps_loss_ref_vs_autograd():
    from oracle import keypoints as okp
    g = torch.Generator().manual_seed(6)
    D, S, K, ld = 3, 4, 2, 16
    low = torch.randn((D, S, S, ld), generator=g) * 3
    loc = torch.randint(0, 16 * S * S, (D, K), generator=g, dtype=torch.int32)
    w = torch.tensor([[1.0, 0.0], [2.0, 1.0], [1.0, 1.0]])
    tw = float(w.sum())
    grad, loss, _ = kps_loss_ref(low, K, loc, w, tw, 0.7, ld)
    lo = low.clone().requires_grad_(True)
    up = okp.bilinear_upsample2x(unpack_low(lo, K))
    lp = F.log_softmax(up.reshape(D * K, -1).double(), dim=1)
    nll = -lp[torch.arange(D * K), loc.reshape(-1).long()]
    ref_loss = (nll * w.reshape(-1).double()).sum() / tw * 0.7
    ref_loss.backward()
    # the oracle's deconv runs in fp32: agreement to its rounding
    assert abs(float(loss.sum()) - float(ref_loss)) <= 1e-5 * abs(float(ref_loss))
    assert float((grad.float() - lo.grad).abs().max()) <= 1e-6 * float(lo.grad.abs().max())
    assert not grad[..., 4 * K:].any() and torch.equal(pack_low(unpack_low(low, K), ld)[..., :4 * K], low[..., :4 * K])
    assert not kps_loss_ref(low, K, loc, w, 0.0, 0.7, ld)[0].any()


def test_sgd_ref_vs_torch_sgd():
    """torch.optim.SGD (momentum buffer b, w -= lr b, b = mu b + g + wd w) is Caffe2's update with m = lr b."""
    g = torch.Generator().manual_seed(7)
    w0 = torch.randn(50, generator=g, dtype=torch.float64)
    gr = torch.randn(50, generator=g, dtype=torch.float64)
    m0 = torch.randn(50, generator=g, dtype=torch.float64) * 0.01
    lr, mu, wd = f32(0.02), f32(0.9), f32(1e-4)
    for lr_mult, wd_mult in ((1.0, 1.0), (2.0, 0.0)):
        p = torch.nn.Parameter(w0.clone())
        opt = torch.optim.SGD([p], lr=lr * lr_mult, momentum=mu, weight_decay=wd * wd_mult)
        opt.state[p]['momentum_buffer'] = m0.clone() / (lr * lr_mult)
        p.grad = gr.clone()
        opt.step()
        nw, nm, bw, bm = sgd_ref(w0, gr, m0, lr, mu, wd, 1.0, lr_mult, wd_mult)
        assert torch.allclose(nw, p.detach(), rtol=1e-14, atol=1e-15)
        assert torch.allclose(nm, opt.state[p]['momentum_buffer'] * lr * lr_mult, rtol=1e-12, atol=1e-16)
        assert bool((bw > 0).all() and (bw < 1e-6 * (nw.abs() + 1)).all())
