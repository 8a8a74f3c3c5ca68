"""GPU: every launch key of the non-GEMM training kernels of csrc/train_ops.cu on the benchmarked training steps (the losses
dt_rpn_loss_grad / dt_frcnn_loss_grad / dt_kps_loss_grad, the joins dt_bwd_pointwise(2) / dt_upsample_add_bwd /
dt_scatter_stride2 / dt_embed_frame / dt_grad_join_f32, dt_subpixel_grad_fix, dt_bias_grad and dt_sgd_update_multi),
launched at the step's shapes on seeded data with edge values and compared element by element with the references of
tests/test_train_reference.py; a coverage test that proves the table lists every key KeypointRcnnTrainer.step (as
`bench.py --train` builds it, and through step_clips at two drawn scales, one clip flipped) and RpnTrainer.step
(`--train-trunk`) launch; and a teacher-forced capture of one bench step that checks every such launch on its own inputs.

The joins, the sub-pixel fix-up and the re-emitted bf16 filters must be bit-identical to their exact emulations; the losses,
the bias gradient and the fp32 master weights must lie inside the per-element bounds derived next to each reference."""
import collections

import numpy as np
import pytest
import torch

from test_train_reference import (bias_grad_bound, bwd_pointwise_ref, embed_frame_ref, f32, frcnn_bounds, frcnn_loss_ref,
                                  grad_join_ref, kps_bounds, kps_loss_ref, pack_low, rpn_grad_bound, rpn_loss_bound,
                                  rpn_loss_ref, rpn_loss_terms, scatter_stride2_ref, sgd_ref, subpixel_fix_ref,
                                  upsample_add_bwd_ref, U24)

pytestmark = pytest.mark.gpu

# ------------------------------------------------------------------ the launch table
# The bench step: R-50-FPN-3D on an 800 x 1344 blob, B = 2 clips of T = 3 frames; res3..res5 = 4, 6, 3 bottleneck blocks
# (res2 frozen); FPN P2..P5 = 200 x 336 .. 25 x 42 (256 channels), P6 = 13 x 21; RPN A = 3 anchors, rows padded to 16;
# box head 2 x 512 RoIs, 2 classes (ld 16); keypoint head 2 x 128 RoIs, 14 x 14 low-res maps, K = 17 joints (ld 72).
RPN_LOSS = {(3, 16, 16, True)}                                   # (A, ld_o, ld_g, loss given)
FRCNN = {(2, 16, 16, 1024, True, True)}                          # (C, ld_o, ld_g, rows, loss given, accuracy given)
KPS = {(14, 17, 72, 72, 256, True)}                              # (S, K, ld, ld_g, D, loss given)
SUBPIXEL = {(17, 512, 72, True)}                                 # (K, Cin, ldc, bias gradient given)
# (g2 given, y given, scale given, C): the RPN conv's ReLU; P5's join with the P6 scatter; branch2b / 2a per stage (inner
# 128, 256, 512); a stage boundary's join of the two input-gradient parts (C3 512, C4 1024); the keypoint convs and fc6 / fc7
POINTWISE = {(False, True, False, 256), (True, False, False, 256), (False, True, True, 128), (False, True, True, 256),
             (False, True, True, 512), (True, False, False, 512), (True, False, False, 1024), (False, True, False, 512),
             (False, True, False, 1024)}
# (g2 given, y given, scale given, scale2 given, C): a block's output gradient for branch2c and the shortcut; g2 is absent for
# the last res5 block (the first of the backward), scale2 present for the first block of each stage (the projection shortcut)
POINTWISE2 = {(False, True, True, False, 2048), (True, True, True, False, 2048), (True, True, True, True, 2048),
              (True, True, True, False, 1024), (True, True, True, True, 1024), (True, True, True, False, 512),
              (True, True, True, True, 512)}
UPSAMPLE = {(True, 256)}                                         # (coarse_in given, C)
# (H odd, W odd, C): P6's gradient onto P5's 25 x 42; the stride-2 1x1 convs' input gradients onto C3 (100 x 168) and C4
SCATTER = {(1, 0, 256), (0, 0, 512), (0, 0, 1024)}
EMBED = {(3, 0)}                                                 # (T, the slice-center frame VIDEO.NUM_FRAMES_MID // 2)
JOIN = {(True,)}                                                 # (bf16 gradient given)
BIAS = {(256, 256), (16, 16), (1024, 1024), (512, 512), (72, 72)}        # (C, ld)
# (items): one per filter and one per bias.  Trunk: 13 blocks x 3 convs + 3 shortcuts = 42 filters, 4 lateral + 4 post FPN
# convs, the RPN conv and the RPN output conv with biases: 42 + 2 * 10 = 62.  Keypoint R-CNN adds fc6, fc7, cls/bbox, the 8
# keypoint convs and kps_score_lowres, all with biases: 62 + 2 * 12 = 86.
SGD = {(86,), (62,)}
TABLE = dict(dt_rpn_loss_grad=RPN_LOSS, dt_frcnn_loss_grad=FRCNN, dt_kps_loss_grad=KPS, dt_subpixel_grad_fix=SUBPIXEL,
             dt_bwd_pointwise=POINTWISE, dt_bwd_pointwise2=POINTWISE2, dt_upsample_add_bwd=UPSAMPLE, dt_scatter_stride2=SCATTER,
             dt_embed_frame=EMBED, dt_grad_join_f32=JOIN, dt_bias_grad=BIAS, dt_sgd_update_multi=SGD)

# launches of one bench step: an RPN loss per level P2..P6; the slice-center embedding per FPN level P5..P2; the top-down
# join at P4, P3, P2; one pointwise2 per res3..res5 block (4 + 6 + 3); one fused SGD launch
STEP_COUNTS = dict(dt_rpn_loss_grad=5, dt_embed_frame=4, dt_upsample_add_bwd=3, dt_bwd_pointwise2=13, dt_sgd_update_multi=1)


def launch_key(name, a):
    """The table key of one L.call(name, *a) of these entry points, or None for other entry points."""
    g = lambda i: a[i] is not None
    if name == 'dt_rpn_loss_grad':
        return (a[7], a[1], a[12], g(13))
    if name == 'dt_frcnn_loss_grad':
        return (a[7], a[1], a[12], a[6], g(13), g(14))
    if name == 'dt_kps_loss_grad':
        return (a[2], a[3], a[1], a[10], a[4], g(11))
    if name == 'dt_subpixel_grad_fix':
        return (a[2], a[3], a[4], g(1))
    if name == 'dt_bwd_pointwise':
        return (g(1), g(2), g(3), a[5])
    if name == 'dt_bwd_pointwise2':
        return (g(1), g(2), g(3), g(7), a[5])
    if name == 'dt_upsample_add_bwd':
        return (g(1), a[5])
    if name == 'dt_scatter_stride2':
        return (a[4] & 1, a[5] & 1, a[6])
    if name == 'dt_embed_frame':
        return (a[2], a[4])
    if name == 'dt_grad_join_f32':
        return (g(0),)
    if name == 'dt_bias_grad':
        return (a[2], a[3])
    if name == 'dt_sgd_update_multi':
        return (a[2],)
    return None


def _bench_cfg():
    import bench
    cfg = bench.bench_cfg(800, 1333, 'r50fpn3d')
    cfg.TRAIN.BATCH_SIZE_PER_IM = 512; cfg.TRAIN.RPN_PRE_NMS_TOP_N = 2000
    return cfg


@pytest.fixture(scope='module')
def step_env():
    """The trainer `bench.py --train` builds, its frames and ground truth."""
    import bench
    from detectandtrack_b200.modeling import params as Pm
    from detectandtrack_b200.modeling.trainer import KeypointRcnnTrainer, pack_gt
    cfg = _bench_cfg()
    blobs, spec = Pm.random_blobs(cfg)
    tr = KeypointRcnnTrainer(cfg, blobs, spec)
    frames = torch.from_numpy(bench.synth_frames(2, 3, 800, 1333, 100)).cuda()
    yield dict(cfg=cfg, blobs=blobs, spec=spec, tr=tr, frames=frames, gt=pack_gt(bench.synth_gt(2, 800, 1333, 7)))
    from test_gpu_engine import _cfg
    _cfg()


def _num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_step_train_ops_are_all_in_the_table(record_property):
    """One KeypointRcnnTrainer.step as bench.py --train runs it, one step_clips of an 800 x 1333 clip at scale 800 and a
    mirrored 720 x 1280 clip drawn to 640 (TRAIN.AUGMENT), and one RpnTrainer.step as --train-trunk runs it: every launch of
    these entry points has a key in TABLE (each with a value test below), and the bench step launches what its graph says."""
    import step_launches as sl
    missing, seen = {}, set()
    for tag in ('train', 'augment', 'trunk'):
        launched = [(name, k) for name, a, _ in sl.record(tag).calls if (k := launch_key(name, a)) is not None]
        if tag == 'train':
            counts = collections.Counter(n for n, _ in launched)
            assert {n: counts[n] for n in STEP_COUNTS} == STEP_COUNTS, dict(counts)
            assert set(counts) == set(TABLE), set(TABLE) - set(counts)
        for name, k in launched:
            seen.add((name, k))
            if k not in TABLE[name]:
                missing.setdefault((name, k), tag)
        record_property('launches_%s' % tag, len(launched))
    record_property('keys_seen', len(seen))
    for s in sorted(seen, key=str):
        print('  ', s)
    assert not missing, missing


# ------------------------------------------------------------------ value tests
def _bf16_bits(t):
    return t.contiguous().view(torch.int16)


def _exact(got, exp, what):
    assert got.shape == exp.shape, (what, got.shape, exp.shape)
    bad = _bf16_bits(got) != _bf16_bits(exp) if got.dtype == torch.bfloat16 else got != exp
    assert not bool(bad.any()), (what, int(bad.sum()), bad.nonzero()[:5].tolist())


def _within(got, ref, bound, what, rec=None):
    err = (got.double() - ref).abs()
    ratio = float((err / bound.clamp_min(1e-300)).max()) if err.numel() else 0.0
    if rec is not None:
        rec('max_err_over_bound_%s' % what, ratio)
    bad = ~(err <= bound)
    assert not bool(bad.any()), (what, int(bad.sum()), bad.nonzero()[:5].tolist(), ratio)
    return ratio


SENT = -12345.0                   # pre-fill of output buffers: every element the kernel should write is checked

# rows of the step's largest tensor of each channel count: P2 RPN rows (256), res3 (128 inner, 512 out), res4 out (1024),
# res5 out (2048)
ROWS_OF_C = {128: 2 * 3 * 100 * 168, 256: 2 * 200 * 336, 512: 2 * 3 * 100 * 168, 1024: 2 * 3 * 50 * 84, 2048: 2 * 3 * 25 * 42}


def _edge_rows(g1, g2, y):
    """Edge values in the first rows: y = +0, -0, the smallest positive bf16 subnormal, NaN, -1 and 1 in turn; g1 + g2
    cancelling exactly; masked sums on bf16 rounding ties (1 + 2^-7 + 2^-8 -> 1 + 2^-6, 1 + 2^-8 -> 1)."""
    C = g1.shape[1]
    ys = torch.tensor([0.0, -0.0, 2.0 ** -133, float('nan'), -1.0, 1.0]).bfloat16().cuda()
    if y is not None:
        y[:4] = ys.repeat(C // 6 + 1)[:C]
        y[4:8] = 1.0
    if g2 is not None:
        g2[4] = -g1[4]
        g1[5], g2[5] = 1 + 2 ** -7, 2 ** -8
        g1[6], g2[6] = 1.0, 2 ** -8
        g1[7], g2[7] = -(1 + 2 ** -7), -2 ** -8


@pytest.mark.parametrize('key', sorted(POINTWISE) + sorted(POINTWISE2), ids=lambda k: '-'.join(str(int(v)) for v in k))
def test_bwd_pointwise_step_shape_bit_exact(key):
    """dt_bwd_pointwise(2) on the step's largest tensor of that width: bit-identical to bwd_pointwise_ref.  Channel scales
    1 and 2 on the first 16 channels keep the masked sums' ties through the product."""
    from detectandtrack_b200.ops import train_ops as to
    second = len(key) == 5
    has_g2, has_y, has_s = key[:3]
    has_s2 = second and key[3]
    Cc = key[-1]
    rows = ROWS_OF_C[Cc]
    g = torch.Generator(device='cuda').manual_seed(Cc + 7 * sum(key[:-1]))
    rnd = lambda: torch.randn((rows, Cc), generator=g, device='cuda').bfloat16()
    g1, g2, y = rnd(), rnd() if has_g2 else None, rnd() if has_y else None
    _edge_rows(g1, g2, y)

    def sc():
        s = torch.rand(Cc, generator=g, device='cuda') + 0.5
        s[:8], s[8:16] = 1.0, 2.0
        return s
    scale, scale2 = sc() if has_s else None, sc() if has_s2 else None
    if second:
        out, out2 = to.bwd_pointwise(g1, g2, y, scale, second=True, scale2=scale2)
        e1, e2 = bwd_pointwise_ref(g1, g2, y, scale, second=True, scale2=scale2)
        _exact(out2, e2, 'out2')
    else:
        out = to.bwd_pointwise(g1, g2, y, scale)
        e1 = bwd_pointwise_ref(g1, g2, y, scale)
    _exact(out, e1, 'out')


def test_upsample_add_bwd_step_shape_bit_exact():
    """The P3 -> P2 top-down join at the step's shape (fine [2, 3, 200, 336, 256]): bit-identical to the emulation, with
    children of magnitudes 2^24, 2^16, 1, 1 where the kernel's order rounds to 2^24 and a pairwise order to 2^24 + 2^17."""
    from detectandtrack_b200.ops import train_ops as to
    g = torch.Generator(device='cuda').manual_seed(21)
    fine = torch.randn((2, 3, 200, 336, 256), generator=g, device='cuda').bfloat16()
    coarse = torch.randn((2, 3, 100, 168, 256), generator=g, device='cuda').bfloat16()
    quad = torch.tensor([[2.0 ** 24, 2.0 ** 16], [1.0, 1.0]]).bfloat16().cuda()
    for i in range(40):
        n, t, h, w, c = i % 2, i % 3, 7 * i % 100, 5 * i % 168, 8 * i % 256
        q = quad if i % 4 < 2 else quad.flip(0, 1)
        fine[n, t, 2 * h:2 * h + 2, 2 * w:2 * w + 2, c] = q * 2.0 ** (i % 9 - 4)
        coarse[n, t, h, w, c] = 0.0 if i % 2 else 2.0 ** (i % 9 - 4)
    out = to.upsample_add_bwd(fine, coarse)
    exp = upsample_add_bwd_ref(fine, coarse)
    _exact(out, exp, 'upsample_add')
    assert float(exp[0, 0, 0, 0, 0]) == 2.0 ** 20           # exact sum 2^20 + 2^12 + 3 * 2^-4 rounds to 2^20 + 2^13


SCATTER_SHAPES = {(1, 0, 256): (2, 25, 42), (0, 0, 512): (6, 100, 168), (0, 0, 1024): (6, 50, 84)}     # (frames, H, W)


@pytest.mark.parametrize('key', sorted(SCATTER), ids=lambda k: '-'.join(map(str, k)))
def test_scatter_stride2_step_shape_exact(key):
    """P6's gradient [2, 13, 21, 256] onto P5's 25 x 42 (odd height: the last row is cropped) and the stride-2 1x1 convs'
    input gradients onto C3 / C4, into buffers pre-filled with a sentinel: every element equals the reference."""
    from detectandtrack_b200 import _lib as L
    Fr, H, W = SCATTER_SHAPES[key]
    Cc = key[2]
    Hs, Ws = (H + 1) // 2, (W + 1) // 2
    g = torch.Generator(device='cuda').manual_seed(22)
    src = torch.randn((Fr, Hs, Ws, Cc), generator=g, device='cuda').bfloat16()
    out = torch.full((Fr, H, W, Cc), SENT, dtype=torch.bfloat16, device='cuda')
    L.call('dt_scatter_stride2', L.ptr(src), Fr, Hs, Ws, H, W, Cc, L.ptr(out), L.stream_ptr())
    _exact(out, scatter_stride2_ref(src, H, W), 'scatter')


@pytest.mark.parametrize('key', sorted(EMBED), ids=lambda k: '-'.join(map(str, k)))
def test_embed_frame_step_shape_exact(key):
    """The slice-center embedding of every FPN level's gradient [2, 1, h, w, 256] into [2, 3, h, w, 256], pre-filled with
    a sentinel: frame c is the source, every other frame zero."""
    from detectandtrack_b200 import _lib as L
    T, c = key
    g = torch.Generator(device='cuda').manual_seed(22)
    for h, w in ((25, 42), (50, 84), (100, 168), (200, 336)):
        s = torch.randn((2, 1, h, w, 256), generator=g, device='cuda').bfloat16()
        full = torch.full((2, T, h, w, 256), SENT, dtype=torch.bfloat16, device='cuda')
        L.call('dt_embed_frame', L.ptr(s), 2, T, h * w * 256, c, L.ptr(full), L.stream_ptr())
        _exact(full, embed_frame_ref(s[:, 0], T, c), 'embed %dx%d' % (h, w))


def test_grad_join_step_shape_bit_exact():
    """The RoI heads' fp32 P2 accumulator [2, 200, 336, 256] joined with the RPN's bf16 gradient: bf16(acc + g)."""
    from detectandtrack_b200.ops import train_ops as to
    g = torch.Generator(device='cuda').manual_seed(23)
    acc = torch.randn((2, 200, 336, 256), generator=g, device='cuda') * 1e-3
    acc[0, 0, 0, :4] = torch.tensor([2 ** -8, -(2 ** -8), 0.0, 2 ** -133], device='cuda')
    gb = torch.randn((2, 200, 336, 256), generator=g, device='cuda').bfloat16()
    gb[0, 0, 0, :4] = torch.tensor([1.0, -1.0, -0.0, 0.0]).bfloat16().cuda()
    _exact(to.grad_join_f32(acc, gb), grad_join_ref(acc, gb), 'join')


def test_subpixel_grad_fix_step_shape_exact():
    """kps_score_lowres' gradient [9, 72, 512] and bias gradient [72] (K = 17): dead taps zero, live taps unchanged, each
    bias quadruple replaced by its fp32 sum ((b0 + b1) + b2) + b3, channels 68..71 zero."""
    from detectandtrack_b200.ops import train_ops as to
    g = torch.Generator(device='cuda').manual_seed(24)
    gW = torch.randn((9, 72, 512), generator=g, device='cuda')
    gb = torch.randn(72, generator=g, device='cuda') * torch.logspace(-6, 6, 72, device='cuda')      # sums where order matters
    ew, eb = subpixel_fix_ref(gW.clone(), gb.clone(), 17)
    to.subpixel_grad_fix(gW, gb, 17)
    _exact(gW, ew, 'gW')
    _exact(gb, eb, 'gb')


def _rpn_problem(rows, A, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    beta = f32(1.0 / 9.0)
    out = torch.randn((rows, 16), generator=g, device='cuda') * 3
    labels = torch.randint(-1, 2, (rows, A), generator=g, device='cuda', dtype=torch.int32)
    tgt = out[:, A:5 * A] + (torch.rand((rows, 4 * A), generator=g, device='cuda') - 0.5) * 0.5
    iw = (torch.rand((rows, 4 * A), generator=g, device='cuda') > 0.3).float()
    ow = torch.where(torch.rand((rows, 4 * A), generator=g, device='cuda') > 0.2, 1.0 / 256, 0.0)
    # logits 0, +-1e-3, +-17, +-90 (expf(-x) overflows at -90) under both labels
    xs = torch.tensor([0.0, 1e-3, -1e-3, 17.0, -17.0, 90.0, -90.0], device='cuda')
    for lab in (0, 1):
        out[lab * 7:(lab + 1) * 7, :A] = xs[:, None]
        labels[lab * 7:(lab + 1) * 7] = lab
    # |d| at beta and one ulp on either side, both signs, with unit inside weights
    b = torch.tensor([beta], dtype=torch.float32)
    ds = torch.cat([torch.nextafter(b, torch.zeros(1)), b, torch.nextafter(b, torch.ones(1))]).cuda()
    ds = torch.cat([ds, -ds])
    out[20:26, A:5 * A] = ds[:, None]
    tgt[20:26] = 0.0
    iw[20:26] = 1.0
    ow[20:26] = 1.0 / 256
    return out.contiguous(), labels, tgt.contiguous(), iw, ow, beta


def _check_rpn(out, labels, tgt, iw, ow, rows, A, s_cls, s_box, beta, grad, ld_g, loss0, loss, rec=None):
    gr = grad.view(rows, ld_g)
    gc, gb, lc, lb = rpn_loss_ref(out, labels, tgt, iw, ow, A, s_cls, s_box, beta)
    bound = rpn_grad_bound(out, labels, tgt, iw, ow, A, s_cls, s_box, beta)
    r = _within(gr[:, :5 * A], torch.cat([gc, gb], 1), bound, 'rpn_grad', rec)
    assert not bool(gr[:, 5 * A:].float().any()) and not bool(gr[:, :A][labels < 0].float().any())
    terms = rpn_loss_terms(out, labels, tgt, iw, ow, A, s_cls, s_box, beta)
    for i, (v, tt) in enumerate(((lc, terms[:, :A]), (lb, terms[:, A:]))):
        bd = rpn_loss_bound(tt, float(loss0[i]), rows, ld_g, _num_sms())
        assert abs(float(loss[i]) - (float(loss0[i]) + v)) <= bd, (i, float(loss[i]), float(loss0[i]) + v, bd)
    return r


def test_rpn_loss_grad_step_shape(record_property):
    """dt_rpn_loss_grad on all 134 400 P2 rows (2 x 200 x 336, A = 3, ld 16) with the step's scales, edge logits, |d| one ulp
    on each side of beta, ignored anchors, onto a nonzero loss: gradient per element within rpn_grad_bound, padding and
    ignored anchors exactly zero (the buffer is pre-filled), both loss sums within rpn_loss_bound."""
    from detectandtrack_b200 import _lib as L
    rows, A, ld = 2 * 200 * 336, 3, 16
    out, labels, tgt, iw, ow, beta = _rpn_problem(rows, A, 25)
    s_cls, s_box = 1.0 / 256 / 2, 1.0 / 2
    grad = torch.full((rows, ld), SENT, dtype=torch.bfloat16, device='cuda')
    loss0 = torch.tensor([0.5, 0.25], device='cuda')
    loss = loss0.clone()
    L.call('dt_rpn_loss_grad', L.ptr(out), 16, L.ptr(labels), L.ptr(tgt), L.ptr(iw), L.ptr(ow), rows, A, s_cls, s_box, beta,
           L.ptr(grad), ld, L.ptr(loss), L.stream_ptr())
    torch.cuda.synchronize()
    _check_rpn(out, labels, tgt, iw, ow, rows, A, s_cls, s_box, beta, grad, ld, loss0.cpu(), loss.cpu(), record_property)


def _frcnn_problem(rows, C, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    out = torch.randn((rows, 16), generator=g, device='cuda') * 3
    labels = torch.randint(0, C, (rows,), generator=g, device='cuda', dtype=torch.int32)
    labels[torch.rand(rows, generator=g, device='cuda') < 0.25] = -1
    tgt = torch.randn((rows, 4 * C), generator=g, device='cuda') * 2
    iw = torch.zeros((rows, 4 * C), device='cuda')
    fg = labels > 0
    iw[fg, 4:8] = 1.0
    ow = iw.clone()
    out[0:4, :C] = 1.5                                    # exact ties: the first class wins (3 hits; the last would give 1)
    labels[0:4] = torch.tensor([0, 0, 0, 1], dtype=torch.int32)
    out[4:8, :C] = torch.tensor([[100.0, -100.0], [-100.0, 100.0], [88.0, -88.0], [-90.0, 90.0]], device='cuda')   # saturated
    labels[4:8] = torch.tensor([0, 0, 1, 1], dtype=torch.int32)
    one = torch.ones(1)
    ds = torch.cat([torch.nextafter(one, torch.zeros(1)), one, torch.nextafter(one, 2 * one)]).cuda()
    ds = torch.cat([ds, -ds])                                                 # |d| at 1 and one ulp on either side
    labels[8:14] = 1
    out[8:14, C + 4:C + 8] = ds[:, None]
    tgt[8:14] = 0.0
    iw[8:14], ow[8:14] = 0.0, 0.0
    iw[8:14, 4:8], ow[8:14, 4:8] = 1.0, 1.0
    return out, labels, tgt.contiguous(), iw, ow


def _check_frcnn(out, labels, tgt, iw, ow, C, N, s_cls, s_box, grad, ld_g, loss0, loss, acc0, acc, rows, rec=None):
    ref, lc, lb, hit = frcnn_loss_ref(out, labels, tgt, iw, ow, C, N, s_cls, s_box)
    gb, b_lc, b_lb = frcnn_bounds(out, labels, tgt, iw, ow, C, N, s_cls, s_box)
    gr = grad.view(rows, ld_g)
    r = _within(gr[:, :5 * C], ref, gb, 'frcnn_grad', rec)
    assert not bool(gr[:, 5 * C:].float().any())
    assert float(acc) == float(acc0) + int(hit.sum()), (float(acc), float(acc0), int(hit.sum()))
    depth = 5 + -(-rows // 32) + 1                       # shuffle tree, one atomicAdd per warp in any order
    for i, (v, b) in enumerate(((lc, b_lc), (lb, b_lb))):
        tot = float(v.sum())
        bd = float(b.sum()) + depth * U24 * (abs(float(loss0[i])) + float(v.abs().sum()))
        assert abs(float(loss[i]) - float(loss0[i]) - tot) <= bd, (i, float(loss[i]), float(loss0[i]) + tot, bd)
    return r


def test_frcnn_loss_grad_step_shape(record_property):
    """dt_frcnn_loss_grad on the step's 1024 RoIs (2 classes, ld 16) with exact logit ties, saturated logits, |d| one ulp on
    each side of 1 and padding rows: gradient within frcnn_bounds per element, padding channels exactly zero, the accuracy
    count exact (first maximum on ties), both loss sums bounded; then totals[0] = 0: every row zero, nothing accumulated."""
    from detectandtrack_b200 import _lib as L
    rows, C, ld = 1024, 2, 16
    out, labels, tgt, iw, ow = _frcnn_problem(rows, C, 26)
    N = float(int((labels >= 0).sum()))
    for n in (N, 0.0):
        totals = torch.tensor([n, 0.0], device='cuda')
        grad = torch.full((rows, ld), SENT, dtype=torch.bfloat16, device='cuda')
        loss0, acc0 = torch.tensor([0.3, 0.2], device='cuda'), torch.tensor([5.0], device='cuda')
        loss, acc = loss0.clone(), acc0.clone()
        L.call('dt_frcnn_loss_grad', L.ptr(out), 16, L.ptr(labels), L.ptr(tgt), L.ptr(iw), L.ptr(ow), rows, C, L.ptr(totals), 1.0, 1.0,
               L.ptr(grad), ld, L.ptr(loss), L.ptr(acc), L.stream_ptr())
        torch.cuda.synchronize()
        _check_frcnn(out, labels, tgt, iw, ow, C, n, 1.0, 1.0, grad, ld, loss0.cpu(), loss.cpu(), acc0.cpu(), acc.cpu(), rows,
                     record_property if n else None)
        if n == 0:
            assert not bool(grad.float().any()) and torch.equal(loss, loss0) and torch.equal(acc, acc0)


def _kps_problem(D, K, S, seed):
    """low [D, S, S, 72] packed: smooth random maps, then crafted RoIs: d = 0 targets on the map's corners, edges and both
    sides of sub-pixel seams; d = 1 a flat map; d = 2 one logit 80 above the rest at the target (p_t -> 1); weights 0, 1, 2."""
    g = torch.Generator().manual_seed(seed)
    S2, M = 2 * S, 4 * S
    m = torch.nn.functional.avg_pool2d(torch.randn((D, K, S2, S2), generator=g), 3, 1, 1) * 3
    loc = torch.randint(0, M * M, (D, K), generator=g, dtype=torch.int32)
    w = torch.randint(0, 3, (D, K), generator=g).float()
    corners = [(0, 0), (0, M - 1), (M - 1, 0), (M - 1, M - 1), (0, 27), (M - 1, 30), (20, 0), (31, M - 1), (27, 28), (28, 27),
               (29, 30), (30, 29), (1, 1), (M - 2, M - 2), (0, 1), (M - 1, M - 2), (13, 14)]
    loc[0] = torch.tensor([y * M + x for y, x in corners[:K]], dtype=torch.int32)
    w[0:3] = 1.0
    m[1] = 0.0                                                              # flat: p = 1 / (4S)^2
    for k in range(K):                                                       # U = u[Y] + u[X]: 240 at (2i, 2i), 160 next
        i = 2 + k % 10
        lv = torch.zeros(S2); lv[i], lv[i + 1] = 160.0, -320.0
        m[2, k] = lv[:, None] + lv[None, :]
        loc[2, k] = (2 * i) * M + 2 * i if k % 2 == 0 else (2 * i + 1) * M + 2 * i
    w[3:8, ::3] = 0.0
    low = pack_low(m, 72).float()
    low[..., 4 * K:] = torch.randn(low[..., 4 * K:].shape, generator=g)     # padding channels are never read
    return low.cuda(), loc.cuda(), w.cuda()


def _check_kps(low, K, loc, w, tw, scale, grad, ld_g, loss0, loss, rec=None):
    ref, lterm, it = kps_loss_ref(low, K, loc, w, tw, scale, ld_g)
    gbound, lbound = kps_bounds(ref, it, ld_g)
    r = _within(grad, ref, gbound, 'kps_grad', rec)
    assert not bool(grad[..., 4 * K:].float().any())
    nat = int(((w > 0) & (tw > 0)).sum())                                    # one atomicAdd per live (RoI, joint), any order
    bd = float(lbound.sum()) + (nat + 1) * U24 * (abs(float(loss0)) + float(lterm.abs().sum()))
    assert abs(float(loss) - float(loss0) - float(lterm.sum())) <= bd, (float(loss), float(loss0) + float(lterm.sum()), bd)
    return r


def test_kps_loss_grad_step_shape(record_property):
    """dt_kps_loss_grad on the step's 256 keypoint RoIs x 17 joints of 14 x 14 low-res maps (ld 72): every gradient element
    within kps_bounds (targets on every corner and edge, across sub-pixel seams, a flat map, a target 80 above the rest,
    zero-weight joints), channels 68..71 zero, the loss sum bounded; then totals[1] = 0: zero gradient, nothing added."""
    from detectandtrack_b200.ops import train_ops as to
    D, K, S = 256, 17, 14
    low, loc, w = _kps_problem(D, K, S, 27)
    tw = float(w.sum())
    for t in (tw, 0.0):
        totals = torch.tensor([0.0, t], device='cuda')
        loss0 = torch.tensor([0.4], device='cuda')
        loss = loss0.clone()
        grad = to.kps_loss_grad(low, K, loc, w, totals, 0.7, 72, loss=loss)
        torch.cuda.synchronize()
        _check_kps(low, K, loc, w, t, f32(0.7), grad, 72, loss0.cpu(), loss.cpu(), record_property if t else None)
        if t == 0:
            assert not bool(grad.float().any()) and torch.equal(loss, loss0)


BIAS_ROWS = {256: 2 * 3 * 200 * 336, 16: 2 * 200 * 336, 1024: 1024, 512: 256 * 14 * 14, 72: 256 * 14 * 14}


@pytest.mark.parametrize('key', sorted(BIAS), ids=lambda k: '%d-%d' % k)
def test_bias_grad_step_shape(key, record_property):
    """dt_bias_grad over the step's largest gradient of that width (P2 of the FPN convs, the RPN output, the FC RoI rows, the
    keypoint maps) onto a nonzero accumulator, within bias_grad_bound per channel."""
    from detectandtrack_b200 import _lib as L
    Cc, ld = key
    rows = BIAS_ROWS[Cc]
    g = torch.Generator(device='cuda').manual_seed(Cc)
    gz = torch.randn((rows, ld), generator=g, device='cuda').bfloat16()
    db0 = torch.randn(Cc, generator=g, device='cuda')
    db = db0.clone()
    L.call('dt_bias_grad', L.ptr(gz), rows, Cc, ld, L.ptr(db), L.stream_ptr())
    torch.cuda.synchronize()
    ref = db0.double() + gz[:, :Cc].double().sum(0)
    _within(db, ref, bias_grad_bound(gz[:, :Cc], db0, rows, _num_sms()), 'bias_%d' % Cc, record_property)


def _sgd_items(tr, n):
    """(w, g, m, w_fwd, w_dgrad, taps, Cout, Cin, lr_mult, wd_mult) of the first n items of the trainer's SGD table, in its
    order (filters, then their biases with 2x lr and no weight decay)."""
    items = []
    for c in tr.convs:
        items.append((c.w, c.g, c.m, c.w_fwd, c.w_dg, c.taps, c.cout, c.cin, 1.0, 1.0))
        if c.bias is not None:
            items.append((c.bias, c.bias_g, c.bias_m, None, None, 1, 1, c.bias.numel(), 2.0, 0.0))
    return items[:n]


def _check_sgd_item(w0, g0, m0, w, m, wf, wdg, lr, mu, wd, gs, lm, wm, what):
    nw, nm, bw, bm = sgd_ref(w0, g0, m0, lr, mu, wd, gs, lm, wm)
    r = max(_within(w, nw, bw, what + ' w'), _within(m, nm, bm, what + ' m'))
    if wf is not None:
        wb = w.view(wf.shape).bfloat16()
        _exact(wf, wb, what + ' w_fwd')
        _exact(wdg, wb.flip(0).transpose(1, 2), what + ' w_dgrad')
    return r


@pytest.mark.parametrize('key', sorted(SGD), ids=lambda k: str(k[0]))
def test_sgd_update_multi_step_table(step_env, key, record_property):
    """dt_sgd_update_multi over copies of every item shape of the bench trainer's table (86 items; the trunk's first 62),
    filters of Cout / Cin 16, 72 and the 1-row biases included, with nonzero momentum, each copy in one flat buffer per
    operand behind a sentinel gap: w and m within sgd_ref's bound, the bf16 forward and dgrad filters equal to bf16(w) and
    its flipped transpose, and every sentinel intact (no item moved twice, nothing outside an item written)."""
    from detectandtrack_b200.ops import train_ops as to
    tr = step_env['tr']
    items = _sgd_items(tr, key[0])
    assert len(items) == key[0]
    gap = 37                                                                     # fp32 / bf16 elements between items
    shapes = [(taps, co, ci, lm, wm) for (_, _, _, wf, _, taps, co, ci, lm, wm) in items]
    total = sum(taps * co * ci + gap for taps, co, ci, _, _ in shapes) + gap
    gen = torch.Generator(device='cuda').manual_seed(28)
    flat = {k: torch.full((total,), SENT, dtype=torch.float32 if k in 'wgm' else torch.bfloat16, device='cuda') for k in ('w', 'g', 'm', 'f', 'd')}
    views, off = [], gap
    for (w, _, _, wf, _, taps, co, ci, lm, wm) in items:
        n = taps * co * ci
        v = {k: flat[k][off:off + n] for k in flat}
        v['w'].copy_(torch.randn(n, generator=gen, device='cuda') * 0.05)
        v['g'].copy_(torch.randn(n, generator=gen, device='cuda') * 1e-2)
        v['m'].copy_(torch.randn(n, generator=gen, device='cuda') * 1e-3)
        views.append((v, wf is not None, off, n))
        off += n + gap
    snap = {k: flat[k].clone() for k in flat}
    bufs = [(v['w'], v['g'], v['m'], v['f'] if hw else None, v['d'] if hw else None) for v, hw, _, _ in views]
    to.sgd_update_multi(to.sgd_table([b + s for b, s in zip(bufs, shapes)]), f32(tr.lr), f32(tr.momentum), f32(tr.wd), 1.0)
    torch.cuda.synchronize()
    worst = 0.0
    mask = torch.ones(total, dtype=torch.bool, device='cuda')
    for (v, hw, o, n), (taps, co, ci, lm, wm) in zip(views, shapes):
        mask[o:o + n] = False
        sh = lambda t: t.view(taps, co, ci)
        worst = max(worst, _check_sgd_item(snap['w'][o:o + n], snap['g'][o:o + n], snap['m'][o:o + n], v['w'], v['m'],
                                           sh(v['f']) if hw else None, v['d'].view(taps, ci, co) if hw else None,
                                           tr.lr, tr.momentum, tr.wd, 1.0, lm, wm, '%dx%dx%d' % (taps, co, ci)))
        if not hw:
            assert bool((v['f'] == SENT).all() and (v['d'] == SENT).all())
    for k in flat:
        _exact(flat[k][mask], snap[k][mask], 'gap ' + k)
        if k == 'g':
            _exact(flat[k], snap[k], 'gradient')
    record_property('max_err_over_bound', worst)


# ------------------------------------------------------------------ teacher-forced capture of a bench step
def _flat(t, n, shape, dtype=None):
    v = t.reshape(-1)
    if dtype is not None and v.dtype != dtype:
        v = v.view(dtype)
    return v[:n].view(shape)


def _cap_rpn(a, get, tr):
    out, ld_o, labels, tgt, iw, ow, rows, A, s_cls, s_box, beta, grad, ld_g, loss = a[:14]
    o = _flat(get(out), rows * ld_o, (rows, ld_o)).clone()
    lab, t = _flat(get(labels), rows * A, (rows, A)).clone(), _flat(get(tgt), rows * 4 * A, (rows, 4 * A)).clone()
    i_w, o_w = _flat(get(iw), rows * 4 * A, (rows, 4 * A)).clone(), _flat(get(ow), rows * 4 * A, (rows, 4 * A)).clone()
    l0 = get(loss)[:2].clone().cpu()
    yield
    return _check_rpn(o, lab, t, i_w, o_w, rows, A, f32(s_cls), f32(s_box), f32(beta), _flat(get(grad), rows * ld_g, (rows, ld_g)), ld_g, l0,
                      get(loss)[:2].cpu())


def _cap_frcnn(a, get, tr):
    out, ld_o, labels, tgt, iw, ow, rows, C_, totals, s_cls, s_box, grad, ld_g, loss, acc = a[:15]
    o = _flat(get(out), rows * ld_o, (rows, ld_o)).clone()
    lab = _flat(get(labels), rows, (rows,)).clone()
    t, i_w, o_w = (_flat(get(x), rows * 4 * C_, (rows, 4 * C_)).clone() for x in (tgt, iw, ow))
    N = float(get(totals)[0])
    l0, a0 = get(loss)[:2].clone().cpu(), get(acc)[:1].clone().cpu()
    yield
    return _check_frcnn(o, lab, t, i_w, o_w, C_, N, f32(s_cls), f32(s_box), get(grad), ld_g, l0, get(loss)[:2].cpu(), a0, get(acc)[:1].cpu(), rows)


def _cap_kps(a, get, tr):
    low, ld, S, K, D, loc, w, totals, scale, grad, ld_g, loss = a[:12]
    lo = _flat(get(low), D * S * S * ld, (D, S, S, ld)).clone()
    lc, wt = _flat(get(loc), D * K, (D, K)).clone(), _flat(get(w), D * K, (D, K)).clone()
    tw = float(get(totals)[1])
    l0 = get(loss)[:1].clone().cpu()
    yield
    return _check_kps(lo, K, lc, wt, tw, f32(scale), _flat(get(grad), D * S * S * ld_g, (D, S, S, ld_g)), ld_g, l0[0], get(loss)[0].cpu())


def _cap_subpixel(a, get, tr):
    gW, gb, K, Cin, ldc = a[:5]
    w0 = _flat(get(gW), 9 * ldc * Cin, (9, ldc, Cin)).clone()
    b0 = _flat(get(gb), ldc, (ldc,)).clone() if gb is not None else None
    ew, eb = subpixel_fix_ref(w0, b0, K)
    yield
    _exact(_flat(get(gW), 9 * ldc * Cin, (9, ldc, Cin)), ew, 'subpixel gW')
    if gb is not None:
        _exact(_flat(get(gb), ldc, (ldc,)), eb, 'subpixel gb')
    return 0.0


def _cap_pointwise(a, get, tr):
    second = len(a) == 10
    g1, g2, y, scale, rows, Cc, out = a[:7]
    bf = lambda p: None if p is None else _flat(get(p), rows * Cc, (rows, Cc)).clone()
    sc = lambda p: None if p is None else _flat(get(p), Cc, (Cc,)).clone()
    args = (bf(g1), bf(g2), bf(y), sc(scale))
    exp = bwd_pointwise_ref(*args, second=True, scale2=sc(a[7])) if second else (bwd_pointwise_ref(*args),)
    yield
    _exact(_flat(get(out), rows * Cc, (rows, Cc)), exp[0], 'pointwise out')
    if second:
        _exact(_flat(get(a[8]), rows * Cc, (rows, Cc)), exp[1], 'pointwise out2')
    return 0.0


def _cap_upsample(a, get, tr):
    fine, coarse, Fr, Hc, Wc, Cc, out = a[:7]
    f = _flat(get(fine), Fr * 4 * Hc * Wc * Cc, (Fr, 2 * Hc, 2 * Wc, Cc))
    c = None if coarse is None else _flat(get(coarse), Fr * Hc * Wc * Cc, (Fr, Hc, Wc, Cc))
    exp = upsample_add_bwd_ref(f, c)
    yield
    _exact(_flat(get(out), Fr * Hc * Wc * Cc, (Fr, Hc, Wc, Cc)), exp, 'upsample_add')
    return 0.0


def _cap_scatter(a, get, tr):
    src, Fr, Hs, Ws, H, W, Cc, out = a[:8]
    exp = scatter_stride2_ref(_flat(get(src), Fr * Hs * Ws * Cc, (Fr, Hs, Ws, Cc)).clone(), H, W)
    yield
    _exact(_flat(get(out), Fr * H * W * Cc, (Fr, H, W, Cc)), exp, 'scatter')
    return 0.0


def _cap_embed(a, get, tr):
    src, B, T, fe, c, out = a[:6]
    exp = embed_frame_ref(_flat(get(src), B * fe, (B, fe)).clone(), T, c)
    yield
    _exact(_flat(get(out), B * T * fe, (B, T, fe)), exp, 'embed')
    return 0.0


def _cap_join(a, get, tr):
    g, acc, n, out = a[:4]
    exp = grad_join_ref(_flat(get(acc), n, (n,)), None if g is None else _flat(get(g), n, (n,)))
    yield
    _exact(_flat(get(out), n, (n,)), exp, 'grad_join')
    return 0.0


def _cap_bias(a, get, tr):
    g, rows, Cc, ld, db = a[:5]
    gz = _flat(get(g), rows * ld, (rows, ld))[:, :Cc].clone()
    d0 = _flat(get(db), Cc, (Cc,)).clone()
    yield
    ref = d0.double() + gz.double().sum(0)
    return _within(_flat(get(db), Cc, (Cc,)), ref, bias_grad_bound(gz, d0, rows, _num_sms()), 'bias')


def _cap_sgd(a, get, tr):
    items = _sgd_items(tr, a[2])
    assert len(items) == a[2]
    lr, mu, wd, gs = a[4:8]
    snap = [(w.clone(), g.clone(), m.clone()) for (w, g, m, *_r) in items]
    yield
    worst = 0.0
    for (w0, g0, m0), (w, g, m, wf, wdg, taps, co, ci, lm, wm) in zip(snap, items):
        _exact(g, g0, 'sgd gradient')
        worst = max(worst, _check_sgd_item(w0, g0, m0, w, m, wf, wdg, lr, mu, wd, gs, lm, wm, '%dx%dx%d' % (taps, co, ci)))
    return worst


CAPTURE = dict(dt_rpn_loss_grad=_cap_rpn, dt_frcnn_loss_grad=_cap_frcnn, dt_kps_loss_grad=_cap_kps, dt_subpixel_grad_fix=_cap_subpixel,
               dt_bwd_pointwise=_cap_pointwise, dt_bwd_pointwise2=_cap_pointwise, dt_upsample_add_bwd=_cap_upsample,
               dt_scatter_stride2=_cap_scatter, dt_embed_frame=_cap_embed, dt_grad_join_f32=_cap_join, dt_bias_grad=_cap_bias,
               dt_sgd_update_multi=_cap_sgd)


def test_teacher_forced_bench_step(step_env, monkeypatch, record_property):
    """One bench KeypointRcnnTrainer.step with every launch of these entry points checked on its own inputs: the inputs
    (in-place ones included: loss accumulators, bias gradients, the sub-pixel gradients, the SGD state) are snapshot,
    the launch runs, and its outputs are compared at once with the references, in the step's real layouts (gradient views
    at unaligned offsets of the flat buffer, padded rows, the heads' accumulator views)."""
    from detectandtrack_b200 import _lib as L
    tr = step_env['tr']
    tensors = {}
    orig_ptr, orig_call = L.ptr, L.call

    def ptr(t):
        if t is not None:
            tensors[t.data_ptr()] = t
        return orig_ptr(t)

    def get(p):
        return None if p is None else tensors[p.value]
    worst, count = {}, collections.Counter()

    def call(name, *a):
        chk = CAPTURE.get(name)
        if chk is None:
            return orig_call(name, *a)
        torch.cuda.synchronize()
        gen = chk(a, get, tr)
        next(gen)
        orig_call(name, *a)
        torch.cuda.synchronize()
        try:
            next(gen)
        except StopIteration as e:
            k = (name,) + launch_key(name, a)
            worst[k] = max(worst.get(k, 0.0), e.value)
            count[k] += 1
    monkeypatch.setattr(L, 'ptr', ptr)
    monkeypatch.setattr(L, 'call', call)
    tr.step(step_env['frames'], step_env['gt'], seed=11)
    torch.cuda.synchronize()
    monkeypatch.undo()
    assert {k[0] for k in count} == set(CAPTURE), set(CAPTURE) - {k[0] for k in count}
    for k, v in sorted(worst.items(), key=str):
        record_property('max_err_over_bound_' + '_'.join(str(x) for x in k), v)
        print('  %s: %d launches, max err / bound %.3g' % (k, count[k], v))
