"""GPU: every filter- and input-gradient launch of the benchmarked training step (tests/test_train_plan.py TRAIN_STEP), at
the reduced shapes that keep the step's plans, bit for bit.

The operands are integers in about [-3, 3] stored in bf16.  Every partial sum of a filter gradient then stays an integer
below 2^24, so fp32 accumulation is exact in any order, split-K reductions included, and the device result must EQUAL the
float64 reference.  The input gradient is an exact fp32 integer rounded once to bf16 in the epilogue, so its bf16 output
must equal bf16(exact sum); magnitudes are picked so that many outputs exceed 256 (where bf16 rounds) and some are exact ties.
Every launch goes through TrainConv.backward, the trainer's own call path."""
import math
import zlib

import numpy as np
import pytest

from test_train_plan import (D_REDUCED, D_ROWS, ROWS, W_REDUCED, W_ROWS, W_FIELDS, dgrad_ref, out_hw, row_dplan, row_wplan,
                             split_ranges, wgrad_key, dgrad_key, wgrad_ref)
from test_train_reference import rpn_loss_ref as _rpn_loss_ref

pytestmark = pytest.mark.gpu


def _seed(name):
    return zlib.crc32(name.encode()) % 100003


def _amplitude(K):
    """Integer operand range [-a, a] for a K-term dgrad sum: each operand has variance a(a+1)/3, so the sum's standard deviation
    is about 600 (well past 256, where bf16 starts to round) and its bound K a^2 stays far below 2^24."""
    a = 3
    while a * (a + 1) / 3.0 < 600.0 / math.sqrt(K):
        a += 1
    return a


def _ints(torch, g, shape, a):
    return torch.randint(-a, a + 1, shape, generator=g).to(torch.bfloat16).cuda()


def _conv(torch, r, seed, wa=3):
    """A TrainConv of the row's shape with integer weights (the bf16 forward / dgrad filters re-emitted by dt_sgd_update_multi
    at lr 0, as the trainer refreshes them), its gradient a view at an 8-byte (not 16-byte) offset of a flat buffer like the
    trainer's, pre-filled with integers."""
    from detectandtrack_b200.modeling.trainer import TrainConv
    from detectandtrack_b200.ops import train_ops as to
    name, N, T, H, W, Cin, Cout, k, s, la, has_bias = r
    rng = np.random.RandomState(seed)
    w = rng.randint(-wa, wa + 1, (Cout, Cin) + tuple(k)).astype(np.float32)
    b = rng.randint(-3, 4, Cout).astype(np.float32) if has_bias else None
    c = TrainConv(torch, w, bias=b, stride=(1,) + tuple(s))
    to.sgd_update(c.w, torch.zeros_like(c.w), torch.zeros_like(c.w), 0.0, 0.0, 0.0, 1.0, c.w_fwd, c.w_dg)
    n = c.w.numel() + (Cout if has_bias else 0)
    flat = torch.from_numpy(rng.randint(-1000, 1001, n + 2).astype(np.float32)).cuda()
    c.g = flat[2:2 + c.w.numel()].view_as(c.w)
    if has_bias:
        c.bias_g = flat[2 + c.w.numel():]
    return c, flat


def _wgrad_failure(r, o, got, exp, gz, x):
    """Worst (tap, Cout tile, Cin tile) with its wrong-entry count, and which split range's contribution the error matches."""
    import torch
    bad = got != exp
    BN = o.BN
    idx = bad.nonzero()
    key = (idx[:, 0] * o.tiles_m + idx[:, 1] // 128) * o.tiles_n + idx[:, 2] // BN
    counts = torch.bincount(key, minlength=o.taps * o.tiles_m * o.tiles_n)
    worst = int(counts.argmax())
    cnt = int(counts[worst])
    t, mt, nt = worst // (o.tiles_m * o.tiles_n), (worst // o.tiles_n) % o.tiles_m, worst % o.tiles_n
    err = (got - exp)[t, mt * 128:(mt + 1) * 128, nt * BN:(nt + 1) * BN].double()
    # contribution of every split range of that unit: position boxes of its k-blocks, tap-shifted input
    N, T, Ho, Wo, _ = gz.shape
    msg = ''
    best = None
    for ks, (k0, k1) in enumerate(split_ranges(o)):
        mask = torch.zeros((N, T, Ho, Wo), dtype=torch.float64, device=gz.device)
        for kb in range(k0, k1):
            iw = kb % o.nW; ih = (kb // o.nW) % o.nH; it = (kb // (o.nW * o.nH)) % o.nT; i_n = kb // (o.nW * o.nH * o.nT)
            mask[i_n * o.TB:(i_n + 1) * o.TB, it * o.TT:(it + 1) * o.TT, ih * o.TH:(ih + 1) * o.TH, iw * o.TW:(iw + 1) * o.TW] = 1
        part = wgrad_ref(gz * mask[..., None].to(gz.dtype), x, r[7], r[8])[t, mt * 128:(mt + 1) * 128, nt * BN:(nt + 1) * BN]
        score = float((err - part).abs().sum().item()), float((err + part).abs().sum().item())
        if best is None or min(score) < best[0]:
            best = (min(score), ks, k0, k1, '+' if score[0] < score[1] else '-')
    if best is not None:
        msg = ', error closest to %s(split range %d = k-blocks [%d, %d), residual %.0f)' % (best[4], best[1], best[2], best[3], best[0])
    return ('%s: %d wrong dW entries; plan %s; worst (tap %d, Cout tile %d, Cin tile %d) with %d%s' %
            (r[0], int(bad.sum()), dict(zip(W_FIELDS, wgrad_key(o))), t, mt, nt, cnt, msg))


@pytest.mark.parametrize('r', W_ROWS, ids=[r[0] for r in W_ROWS])
def test_wgrad_of_every_step_layer_is_exact(r):
    """dW (and db) accumulate into pre-filled buffers: dW == init + sum, bit for bit.  A dropped k-block, a wrong tap shift,
    a padded split range that writes something or a lost split range all change some entry."""
    import torch
    name, _, _, _, _, Cin, Cout, k, s, la, has_bias = r
    N, T, H, W = W_REDUCED[name]
    Ho, Wo = out_hw(H, W, s)
    g = torch.Generator().manual_seed(_seed(name))
    x = _ints(torch, g, (N, T, H, W, Cin), 3)
    gz = _ints(torch, g, (N, T, Ho, Wo, Cout), 3)
    c, flat = _conv(torch, r, 11)
    init = c.g.clone()
    binit = c.bias_g.clone() if has_bias else None
    c.backward(gz, x, need_dx=False)
    torch.cuda.synchronize()
    assert c.g.data_ptr() % 16 == 8
    exp = (init.double() + wgrad_ref(gz, x, k, s)).float()
    o = row_wplan(r, (N, T, H, W))
    if not torch.equal(c.g, exp):
        pytest.fail(_wgrad_failure(r, o, c.g, exp, gz, x))
    if has_bias:
        bexp = (binit.double() + gz.double().reshape(-1, Cout).sum(0)).float()
        assert torch.equal(c.bias_g, bexp), (name, 'db', int((c.bias_g != bexp).sum()))


def test_rpn_convs_accumulate_five_levels_into_one_gradient():
    """The RPN conv and the RPN output conv run once per level (P2..P6) into one dW / db: the sum must be exact."""
    import torch
    for which in ('rpn conv', 'rpn out'):
        rows = [ROWS['%s P%d' % (which, l)] for l in (2, 3, 4, 5, 6)]
        c, _ = _conv(torch, rows[0], 5)
        exp = c.g.double().clone()
        bexp = c.bias_g.double().clone()
        g = torch.Generator().manual_seed(77)
        for r in rows:
            N, T, H, W = W_REDUCED[r[0]]
            x = _ints(torch, g, (N, T, H, W, r[5]), 3)
            gz = _ints(torch, g, (N, T, H, W, r[6]), 3)
            c.backward(gz, x, need_dx=False)
            exp += wgrad_ref(gz, x, r[7])
            bexp += gz.double().reshape(-1, r[6]).sum(0)
        torch.cuda.synchronize()
        assert torch.equal(c.g, exp.float()), (which, int((c.g != exp.float()).sum()))
        assert torch.equal(c.bias_g, bexp.float()), which


def _dgrad_failure(r, o, got, exp):
    N, T, H, W, Cin = got.shape
    bad = (got.float() != exp.float())
    if r[8] != (1, 1):
        return '%s: %d wrong dx entries after the stride-2 scatter; plan %s' % (r[0], int(bad.sum()), dict(zip(('BN', 'TH', 'TW', 'TT', 'TB'), (o.BN, o.TH, o.TW, o.TT, o.TB))))
    import torch
    idx = bad.nonzero()
    dims = (-(-N // o.TB), -(-T // o.TT), -(-H // o.TH), -(-W // o.TW), -(-Cin // o.BN))
    parts = (idx[:, 0] // o.TB, idx[:, 1] // o.TT, idx[:, 2] // o.TH, idx[:, 3] // o.TW, idx[:, 4] // o.BN)
    key = parts[0]
    for d, p in zip(dims[1:], parts[1:]):
        key = key * d + p
    counts = torch.bincount(key)
    worst = int(counts.argmax())
    cnt = int(counts[worst])
    coords = []
    for d in reversed(dims):
        coords.append(worst % d)
        worst //= d
    nb, tb, hb, wb, ct = coords[::-1]
    mt = '(image box %d, frame box %d, row box %d, column box %d)' % (nb, tb, hb, wb)
    return ('%s: %d wrong dx entries; plan BN %d, M tile (TB %d, TT %d, TH %d, TW %d); worst (M tile %s, column tile %d) with %d' %
            (r[0], int(bad.sum()), o.BN, o.TB, o.TT, o.TH, o.TW, mt, ct, cnt))


@pytest.mark.parametrize('r', D_ROWS, ids=[r[0] for r in D_ROWS])
def test_dgrad_of_every_step_layer_is_bf16_of_the_exact_sum(r):
    """dx = conv(gz, w_dg) with bf16 output: bit-identical to bf16(exact sum), i.e. one round to nearest even."""
    import torch
    import torch.nn.functional as F
    name, _, _, _, _, Cin, Cout, k, s, la, has_bias = r
    N, T, H, W = D_REDUCED[name]
    Ho, Wo = out_hw(H, W, s)
    a = _amplitude(Cout * k[0] * k[1] * k[2])
    g = torch.Generator().manual_seed(_seed(name))
    gz = _ints(torch, g, (N, T, Ho, Wo, Cout), a)
    x = torch.zeros((N, T, H, W, Cin), dtype=torch.bfloat16, device='cuda')      # only its shape matters for dx
    c, _ = _conv(torch, r, 13, wa=a)
    dx, _ = c.backward(gz, x, need_dx=True)
    torch.cuda.synchronize()
    wpk = c.w.double()                                                           # [taps, Cout, Cin] integers
    ref = dgrad_ref(gz, wpk, k, (H, W), s)
    assert float(ref.abs().max()) < 2 ** 24
    exp = ref.float().to(torch.bfloat16)
    mag = ref.abs()
    assert int((mag > 256).sum()) >= 0.2 * ref.numel(), (name, 'too few outputs where bf16 rounds')
    # exact ties: odd integers in (256, 512) lie halfway between two bf16 values (round to nearest EVEN decides)
    assert int(((mag > 256) & (mag < 512) & (torch.remainder(mag, 2) == 1)).sum()) >= 100, (name, 'no rounding ties')
    o = row_dplan(r, (N, T, H, W))
    if not torch.equal(dx.view(torch.int16), exp.view(torch.int16)):
        pytest.fail(_dgrad_failure(r, o, dx, exp))
    if s != (1, 1):                                                              # the scatter against autograd of the strided conv
        xx = torch.zeros((N, Cin, T, H, W), dtype=torch.float64, device='cuda', requires_grad=True)
        w5 = c.w.double().reshape(Cout, Cin)[:, :, None, None, None]
        F.conv3d(xx, w5, None, (1,) + tuple(s)).backward(gz.double().permute(0, 4, 1, 2, 3))
        assert torch.equal(dx, xx.grad.permute(0, 2, 3, 4, 1).float().to(torch.bfloat16)), name


# ---------------------------------------------------------------------------------------------------- dt_rpn_loss_grad
def test_rpn_loss_grad_vs_fp64_formulas():
    """SigmoidCrossEntropy + SmoothL1 (beta 1/9) gradients against the fp64 formulas, within the bf16 output bound; ignored
    anchors and the padding channels [5A, ld_g) exactly zero; |d| on both sides of beta; a row count that is not a multiple
    of the block; the loss accumulates over two launches."""
    import torch
    from detectandtrack_b200 import _lib as L
    A, ld_o, ld_g, rows = 3, 16, 16, 1000 * 7 + 13
    beta = 1.0 / 9.0
    s_cls, s_box = 1.0 / 256 / 2, 1.0 / 2
    g = torch.Generator().manual_seed(3)
    out = (torch.randn((rows, ld_o), generator=g) * 3).cuda()
    labels = torch.randint(-1, 2, (rows, A), generator=g, dtype=torch.int32).cuda()
    tgt = (out[:, A:5 * A] + (torch.rand((rows, 4 * A), generator=g).cuda() - 0.5) * 0.5).contiguous()   # |d| straddles beta
    iw = (torch.rand((rows, 4 * A), generator=g) > 0.3).float().cuda()
    ow = torch.where(torch.rand((rows, 4 * A), generator=g) > 0.2, 1.0 / 256, 0.0).float().cuda()
    grad = torch.full((rows, ld_g), 7.0, dtype=torch.bfloat16, device='cuda')
    loss = torch.tensor([0.5, 0.25], dtype=torch.float32, device='cuda')
    for _ in range(2):
        L.call('dt_rpn_loss_grad', L.ptr(out), ld_o, L.ptr(labels), L.ptr(tgt), L.ptr(iw), L.ptr(ow), rows, A, s_cls, s_box, beta,
               L.ptr(grad), ld_g, L.ptr(loss), L.stream_ptr())
    torch.cuda.synchronize()
    gc, gb, lc, lb = _rpn_loss_ref(out, labels, tgt, iw, ow, A, s_cls, s_box, beta)
    d = (iw.double() * (out[:, A:5 * A].double() - tgt.double())).abs()
    assert int((d[iw > 0] < beta).sum()) > 1000 and int((d[iw > 0] > beta).sum()) > 1000
    ref = torch.cat([gc, gb], 1)
    got = grad[:, :5 * A].double()
    bound = 2.0 ** -8 * ref.abs() + 2.0 ** -22 * max(s_cls, s_box)      # bf16 output; fp32 sigmoid next to 1
    assert bool(((got - ref).abs() <= bound).all()), float(((got - ref).abs() / (ref.abs() + 1e-30)).max())
    assert bool((grad[:, :A][labels < 0] == 0).all())
    assert bool((grad[:, 5 * A:] == 0).all())
    got_l = loss.double().cpu()
    exp_l = torch.tensor([0.5 + 2 * lc, 0.25 + 2 * lb], dtype=torch.float64)
    assert torch.allclose(got_l, exp_l, rtol=1e-4, atol=0), (got_l, exp_l)          # fp32 partial sums and atomics


# ---------------------------------------------------------------------------------------------------- coverage
def test_step_launches_only_table_plans_and_keeps_padding_zero():
    """One full-size KeypointRcnnTrainer.step as bench.py builds it: every wgrad launch and every dgrad conv launched from
    TrainConv.backward has a plan key of a TRAIN_STEP row, and after the update the padding filter rows / biases of the
    padded output convs and the dead sub-pixel taps are exactly zero in every copy of the weights (export_blobs relies on
    it)."""
    import collections
    import ctypes as C
    from detectandtrack_b200 import _lib as L
    import step_launches as sl
    rec = sl.record('train')
    wkeys = {wgrad_key(row_wplan(r)) for r in W_ROWS}
    dkeys = {dgrad_key(row_dplan(r)) for r in D_ROWS}
    seen_w, seen_d = collections.Counter(), collections.Counter()
    for name, a, in_backward in rec.calls:
        if name == 'dt_wgrad_nhwc':
            o = L.WgradPlan()
            assert L.lib().dt_wgrad_nhwc_plan(a[1], a[3], *a[4:17], C.byref(o)) == 0, L.lib().dt_last_error()
            seen_w[wgrad_key(o)] += 1
        elif name == 'dt_conv3d' and in_backward:
            seen_d[dgrad_key(sl.conv_plan(a)[1])] += 1
    print('wgrad launches %d (%d plans), dgrad launches %d (%d plans)' % (sum(seen_w.values()), len(seen_w), sum(seen_d.values()), len(seen_d)))
    assert set(seen_w) <= wkeys, set(seen_w) - wkeys
    assert set(seen_d) <= dkeys, set(seen_d) - dkeys
    assert sum(seen_w.values()) == rec.facts['convs'] + 2 * 4          # the two RPN convs run at five levels
    # padding rows / biases and dead sub-pixel taps stay exactly zero in the master, forward and dgrad filters
    for name, (rows, w_nonzero, b_nonzero) in rec.facts['padding'].items():
        assert rows > 0 and w_nonzero == 0 and b_nonzero == 0, name
    assert rec.facts['dead_taps'][0] > 0 and rec.facts['dead_taps'][1] == 0, rec.facts['dead_taps']
