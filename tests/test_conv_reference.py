"""CPU: the fp64 reference the conv value tests (tests/test_gpu_conv.py) compare conv_tc_kernel with.  It is a sum over
filter taps of GEMMs on the zero-padded, tap-shifted input, so it shares nothing with the kernel's implicit GEMM or with
cuDNN, and on the device it runs as DGEMMs, fast enough for problems that fill several waves of the GPU.  Pinned here
once against torch's own fp64 conv3d."""
import torch
import torch.nn.functional as F


def conv_ref(x, w, stride, pad, scale=None, bias=None, residual=None, res_mode=0, relu=False):
    """x [N, T, H, W, Cin], w [Cout, Cin, kT, kH, kW] (any float type, any device) -> fp64 [N, To, Ho, Wo, Cout] =
    relu?(conv(x, w) * scale + bias (+ residual, or its nearest-2x upsample for res_mode 2))."""
    x, w = x.double(), w.double()
    N, T, H, W, Cin = x.shape
    Cout, _, kT, kH, kW = w.shape
    (sT, sH, sW), (pT, pH, pW) = stride, pad
    To, Ho, Wo = (T + 2 * pT - kT) // sT + 1, (H + 2 * pH - kH) // sH + 1, (W + 2 * pW - kW) // sW + 1
    xp = F.pad(x, (0, 0, pW, pW, pH, pH, pT, pT))
    y = torch.zeros((N * To * Ho * Wo, Cout), dtype=torch.float64, device=x.device)
    for kt in range(kT):
        for kh in range(kH):
            for kw in range(kW):
                xs = xp[:, kt:kt + sT * (To - 1) + 1:sT, kh:kh + sH * (Ho - 1) + 1:sH, kw:kw + sW * (Wo - 1) + 1:sW]
                y += xs.reshape(-1, Cin) @ w[:, :, kt, kh, kw].t()
    y = y.view(N, To, Ho, Wo, Cout)
    if scale is not None:
        y = y * scale.double()
    if bias is not None:
        y = y + bias.double()
    if res_mode == 1:
        y = y + residual.double()
    elif res_mode == 2:
        y = y + residual.double().repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)
    return y.clamp_min(0) if relu else y


def test_tap_sum_reference_equals_torch_conv3d():
    g = torch.Generator().manual_seed(5)
    x = torch.randn((2, 4, 11, 13, 6), generator=g)
    w = torch.randn((5, 6, 3, 3, 3), generator=g)
    scale, bias = torch.rand(5, generator=g) + 0.5, torch.randn(5, generator=g)
    for stride, pad in (((1, 1, 1), (1, 1, 1)), ((1, 2, 2), (0, 1, 1)), ((2, 1, 2), (1, 0, 1))):
        y = conv_ref(x, w, stride, pad, scale, bias)
        ref = F.conv3d(x.permute(0, 4, 1, 2, 3).double(), w.double(), None, stride, pad).permute(0, 2, 3, 4, 1)
        ref = ref * scale.double() + bias.double()
        assert y.dtype == torch.float64 and y.shape == ref.shape
        assert (y - ref).abs().max().item() <= 1e-12 * ref.abs().max().item()
    # residual epilogues: same shape, and the nearest-2x upsample of the FPN top-down add, then ReLU
    y = conv_ref(x, w, (1, 1, 1), (1, 1, 1))
    res = torch.randn(y.shape, generator=g)
    assert torch.equal(conv_ref(x, w, (1, 1, 1), (1, 1, 1), residual=res, res_mode=1, relu=True), (y + res.double()).clamp_min(0))
    x2 = torch.randn((1, 2, 8, 6, 6), generator=g)
    y = conv_ref(x2, w, (1, 1, 1), (1, 1, 1))
    top = torch.randn((1, 2, 4, 3, 5), generator=g)
    up = conv_ref(x2, w, (1, 1, 1), (1, 1, 1), residual=top, res_mode=2)
    assert torch.equal(up[:, :, 5, 3], y[:, :, 5, 3] + top[:, :, 2, 1].double())


# ------------------------------------------------------------------ exact forward checks on integer operands
# The forward value tests also run on integer operands (tests/test_gpu_conv.py `operands='integer'`).  In the split modes
# the stored hi and lo halves are independent integers of the same size: not pairs the engine would produce, but the
# kernel's contract is D = x_hi*w_hi + x_lo*w_hi + x_hi*w_lo for any stored pair, and with lo as large as hi each of the
# three products is equally visible.  While the bound on sum |terms| per output stays below 2^22 on a 1/4 grid (powers of
# two for the AffineChannel scale, multiples of 1/4 for the bias), every partial sum is an fp32 value in any order and
# under any truncation inside the MMA, so the device output must equal the emulation below bit for bit.
EXACT_LIMIT = 2 ** 22
INT_LIMIT = {'bf16': 256, 'f16': 2048, 'tf32': 2048}      # integers every value of the operand format holds exactly
SCALES = (0.5, 1.0, 2.0)
BIAS_MAX = 64.0
PRODUCTS = (('x_hi*w_hi', 0, 0), ('x_lo*w_hi', 1, 0), ('x_hi*w_lo', 0, 1))


def int_amplitude(K, fmt='bf16'):
    """Integer operand range [-a, a] for a K-term sum: as test_gpu_train_grads._amplitude (the sum's standard deviation
    about 600, well past 256 where bf16 outputs start to round), within what the operand format holds exactly."""
    a = 3
    while a * (a + 1) / 3.0 < 600.0 / K ** 0.5:
        a += 1
    return min(a, INT_LIMIT[fmt])


def exact_bound(a, K, split, scale_max=max(SCALES), bias_max=BIAS_MAX, res_a=0):
    """Bound on sum |terms| of one output: 3 a^2 K products for split inputs (a^2 K otherwise) times the scale, plus the
    bias and the residual (hi + lo of integers in [-res_a, res_a] for split storage)."""
    return (3 if split else 1) * a * a * K * scale_max + bias_max + (2 if split else 1) * res_a


def _as_f32_bits(v):
    return v.float().contiguous().view(torch.int32)


def round_bf16(v):
    """fp64 of bf16(v), round to nearest even (cvt.rn.bf16.f32) of a value exact in fp32."""
    u = _as_f32_bits(v)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & ~0xFFFF
    return u.view(torch.float32).double()


def round_tf32(v):
    """fp64 of the epilogue's round_to_tf32(v) (conv_tc.cu; cv.round_tf32 on the host), of a value exact in fp32."""
    u = _as_f32_bits(v)
    u = (u + 0xFFF + ((u >> 13) & 1)) & ~0x1FFF
    return u.view(torch.float32).double()


def split_pair(v, fmt):
    """The epilogue's [hi | lo] split: hi = r(v), lo = r(v - hi) with r = bf16 or tf32 rounding (v - hi exact in fp32)."""
    r = round_bf16 if fmt == 'bf16' else round_tf32
    hi = r(v)
    return hi, r(v - hi)


def exact_epilogue(acc, scale=None, bias=None, res=(), relu=False):
    """acc * scale + bias + each residual term, then ReLU, in fp64 (exact under EXACT_LIMIT)."""
    v = acc.double()
    if scale is not None:
        v = v * scale.double()
    if bias is not None:
        v = v + bias.double()
    for r in res:
        v = v + r.double()
    return v.clamp_min(0) if relu else v


def upsample_res(r, res_mode):
    """The residual as the epilogue adds it to an output of the conv's shape (res_mode 2: nearest 2x in H and W)."""
    return r.repeat_interleave(2, dim=2).repeat_interleave(2, dim=3) if res_mode == 2 else r


def exact_store(v, kind):
    """Epilogue value v -> the stored output: 'bf16' rows (round to nearest even), 'bf16 pair' / 'tf32 pair' rows
    [hi | lo], 'f32 tf32' (out_round_tf32) or 'f32' as is."""
    if kind == 'bf16':
        return round_bf16(v).to(torch.bfloat16)
    if kind in ('bf16 pair', 'tf32 pair'):
        fmt = kind.split()[0]
        return torch.cat(split_pair(v, fmt), -1).to(torch.bfloat16 if fmt == 'bf16' else torch.float32)
    if kind == 'f32 tf32':
        return round_tf32(v).float()
    assert kind == 'f32', kind
    return v.float()


def same_bits(a, b):
    """Elementwise: equal bit patterns, with +0 and -0 taken as equal (no consumer of a conv output sees the sign of a
    zero: the next conv, the residual adds, ReLU and the heads' decodes all treat them alike)."""
    assert a.dtype == b.dtype and a.shape == b.shape, (a.dtype, b.dtype, a.shape, b.shape)
    it = torch.int16 if a.element_size() == 2 else torch.int32
    return (a.contiguous().view(it) == b.contiguous().view(it)) | ((a == 0) & (b == 0))


def exact_terms(xs, ws, stride, pad):
    """{product: fp64 conv} of the products the kernel forms: one x*w, or the three of the split modes (never hi + lo)."""
    if len(xs) == 1:
        return {'x*w': conv_ref(xs[0], ws[0], stride, pad)}
    return {n: conv_ref(xs[i], ws[j], stride, pad) for n, i, j in PRODUCTS}


def term_contributions(xs, ws, stride, pad, idx, bk):
    """The contribution of every (tap, k-block of bk channels, product) to the output element idx = (n, t, h, w, c), for
    a failure report: {(tap (kt, kh, kw), k-block, product): fp64 value}, taps whose input lies in the padding left out."""
    n, t, h, w, c = idx
    Cout, Cin, kT, kH, kW = ws[0].shape
    T, H, W = xs[0].shape[1:4]
    prods = (('x*w', 0, 0),) if len(xs) == 1 else PRODUCTS
    out = {}
    for kt in range(kT):
        for kh in range(kH):
            for kw in range(kW):
                ti, hi, wi = t * stride[0] - pad[0] + kt, h * stride[1] - pad[1] + kh, w * stride[2] - pad[2] + kw
                if not (0 <= ti < T and 0 <= hi < H and 0 <= wi < W):
                    continue
                for name, i, j in prods:
                    p = xs[i][n, ti, hi, wi].double() * ws[j][c, :, kt, kh, kw].double()
                    for kb in range(-(-Cin // bk)):
                        out[((kt, kh, kw), kb, name)] = float(p[kb * bk:(kb + 1) * bk].sum())
    return out


def test_rounding_emulations_match_torch_and_the_kernel_formulas():
    """round_bf16 == torch's fp32 -> bf16 conversion (nearest even) on random values and on exact ties of both parities;
    round_tf32 == round to nearest even at 10 mantissa bits (torch.round is half-to-even), on the same kinds of values;
    the pair splits are exact (hi + lo == v where 16 / 22 bits suffice) and round the rest as the epilogue does."""
    g = torch.Generator().manual_seed(9)
    v = torch.randn(100000, generator=g) * 10.0 ** (torch.rand(100000, generator=g) * 12 - 6)
    ints = torch.randint(-2 ** 22, 2 ** 22, (100000,), generator=g).float() / 4
    ties_bf16 = (torch.randint(128, 256, (4096,), generator=g).float() * 2 + 1) * 2.0 ** torch.randint(-10, 10, (4096,), generator=g).float()
    ties_tf32 = (torch.randint(1024, 2048, (4096,), generator=g).float() * 2 + 1) * 2.0 ** torch.randint(-10, 10, (4096,), generator=g).float()
    for x in (v, ints, ties_bf16, -ties_bf16, ties_tf32, -ties_tf32, torch.tensor([0.0, -0.0, 256.0, 257.0, 259.0, -257.0])):
        assert torch.equal(round_bf16(x).float().view(torch.int32), x.to(torch.bfloat16).float().view(torch.int32))
        e = torch.floor(torch.log2(x.double().abs().clamp_min(1e-300)))
        ulp = 2.0 ** (e - 10)
        want = torch.where(x == 0, x.double(), torch.round(x.double() / ulp) * ulp)
        assert torch.equal(round_tf32(x), want)
    assert int((round_bf16(ties_bf16) != ties_bf16.double()).sum()) == ties_bf16.numel()
    for fmt, bits in (('bf16', 16), ('tf32', 22)):
        x = torch.randint(-2 ** (bits - 1), 2 ** (bits - 1), (50000,), generator=g).double()
        hi, lo = split_pair(x, fmt)
        assert torch.equal(hi + lo, x)
        hi, lo = split_pair(ints.double(), fmt)
        assert torch.equal(lo, (round_bf16 if fmt == 'bf16' else round_tf32)(ints.double() - hi))
    # stored outputs: bf16 rows, pairs and tf32-rounded fp32 carry those values
    x = ints.double().view(100, 1000)
    assert torch.equal(exact_store(x, 'bf16').double(), round_bf16(x))
    p = exact_store(x, 'tf32 pair')
    assert p.shape == (100, 2000) and torch.equal(p[:, :1000].double() + p[:, 1000:].double(), x)
    p = exact_store(x, 'bf16 pair').double()
    assert torch.equal(p[:, :1000] + p[:, 1000:], round_bf16(x) + round_bf16(x - round_bf16(x)))
    assert bool(same_bits(torch.tensor([0.0, 1.0]), torch.tensor([-0.0, 1.0])).all())
    assert not bool(same_bits(torch.tensor([1.0]), torch.tensor([-1.0])).any())


def _modes_and_rows():
    from test_conv_plan import R50_FPN_3D, REDUCED, layer_modes
    from test_conv_plan_workloads import STACKED_STRIDED, STACKED_STRIDED_REDUCED, TABLES
    out = [(l, m) for l in R50_FPN_3D for m in layer_modes(l)]
    out += [(l, m) for rows, _, modes in TABLES.values() for l in rows for m in modes(l)]
    out += [(STACKED_STRIDED, m) for m in ('bf16', 'tf32', 'tf32x3', 'bf16x3')]
    return out


def operand_format(mode):
    return {'bf16': 'bf16', 'bf16x3': 'bf16', 'f16': 'f16', 'tf32': 'tf32', 'tf32x3': 'tf32'}[mode]


def test_every_table_row_meets_the_exactness_precondition():
    """For every (row, mode) the forward value tests run on integer operands (test_conv_plan.R50_FPN_3D, the three
    test_conv_plan_workloads tables, the stacked strided case): the operand range holds in the operand format, and the
    bound on sum |terms| per output, with the largest scale, bias and residual, lies below 2^22."""
    n = 0
    for l, m in _modes_and_rows():
        Cin, k, rm = l[5], l[7], l[10]
        K = Cin * k[0] * k[1] * k[2]
        fmt = operand_format(m)
        a = int_amplitude(K, fmt)
        split = m in ('bf16x3', 'tf32x3')
        assert 3 <= a <= INT_LIMIT[fmt], (l[0], m, a)
        assert exact_bound(a, K, split, res_a=a if rm else 0) < EXACT_LIMIT, (l[0], m, a, K)
        n += 1
    assert n > 300


def test_integer_fixture_sees_every_term():
    """A small 3x3x3 proxy conv (Cin 128 = two 64-channel k-blocks) on independent integer hi / lo operands, through the
    emulated bf16-pair epilogue: dropping any single (tap, k-block, product) changes the output, and so do the neighbouring
    arithmetics (lo*lo added, either cross product dropped) in most outputs."""
    g = torch.Generator().manual_seed(3)
    N, T, H, W, Cin, Cout, k, s, p = 2, 3, 5, 6, 128, 8, (3, 3, 3), (1, 1, 1), (1, 1, 1)
    a = int_amplitude(Cin * 27)
    xs = [torch.randint(-a, a + 1, (N, T, H, W, Cin), generator=g).double() for _ in range(2)]
    ws = [torch.randint(-a, a + 1, (Cout, Cin) + k, generator=g).double() for _ in range(2)]
    scale = torch.tensor(SCALES)[torch.randint(0, 3, (Cout,), generator=g)].double()
    bias = torch.randint(-256, 257, (Cout,), generator=g).double() / 4
    terms = exact_terms(xs, ws, s, p)
    acc = sum(terms.values())
    want = exact_store(exact_epilogue(acc, scale, bias), 'bf16 pair')
    n = 0
    for name, i, j in PRODUCTS:
        for kb in range(2):
            for tap in range(27):
                wm = torch.zeros_like(ws[j])
                wm[:, kb * 64:(kb + 1) * 64, tap // 9, tap // 3 % 3, tap % 3] = ws[j][:, kb * 64:(kb + 1) * 64, tap // 9, tap // 3 % 3, tap % 3]
                got = exact_store(exact_epilogue(acc - conv_ref(xs[i], wm, s, p), scale, bias), 'bf16 pair')
                assert not bool(same_bits(got, want).all()), (name, kb, tap)
                n += 1
    assert n == 3 * 2 * 27
    lolo = conv_ref(xs[1], ws[1], s, p)
    for wrong in (acc + lolo, acc - terms['x_lo*w_hi'], acc - terms['x_hi*w_lo']):
        got = exact_store(exact_epilogue(wrong, scale, bias), 'bf16 pair')
        assert float((~same_bits(got, want)).double().mean()) > 0.5
    # the per-element report names the dropped term
    wm = torch.zeros_like(ws[0])
    wm[:, 64:, 1, 2, 0] = ws[0][:, 64:, 1, 2, 0]
    idx = (1, 1, 2, 3, 5)
    c = term_contributions(xs, ws, s, p, idx, 64)
    assert c[((1, 2, 0), 1, 'x_lo*w_hi')] == float(conv_ref(xs[1], wm, s, p)[idx])
    assert sum(c.values()) == float(acc[idx])
