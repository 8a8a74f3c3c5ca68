"""GPU: the Winograd F(2x2, 3x3) path of the bf16x3 keypoint head (csrc/wino.cu, dt_wino_gemm in csrc/conv_tc.cu).

Transforms bit for bit against a numpy emulation of the same fp32 operations; the GEMM against fp64 with a derived bound;
whole layers against the fp64 direct conv; the whole head against the direct path; and which engines take the path."""
import types

import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = pytest.mark.gpu

from detectandtrack_b200.ops import conv as cv        # noqa: E402

S = 14
NT = S // 2


def _bf16(a):
    """fp32 -> the fp32 value of its bf16 rounding (nearest, ties to even)."""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32)


def _split(v):
    hi = _bf16(v)
    return hi, _bf16(v - hi)


def _pairs_to_np(t):
    """bf16 pair tensor [..., 2C] -> (hi, lo) fp32 numpy."""
    a = t.float().cpu().numpy()
    c = a.shape[-1] // 2
    return a[..., :c], a[..., c:]


def _np_to_pairs(hi, lo):
    return torch.from_numpy(np.concatenate([hi, lo], -1)).cuda().to(torch.bfloat16).contiguous()


def _edge_values(rng, shape):
    """fp32 values with signed zeros, values at the ReLU boundary and bf16 rounding ties mixed in."""
    a = rng.randn(*shape).astype(np.float32)
    flat = a.reshape(-1)
    n = flat.size
    idx = rng.randint(0, n, size=(6, max(1, n // 50)))
    flat[idx[0]] = 0.0
    flat[idx[1]] = -0.0
    flat[idx[2]] = -1e-30
    flat[idx[3]] = np.float32(1 + 2 ** -8)             # halfway between two bf16 values
    flat[idx[4]] = np.float32(-(1 + 3 * 2 ** -8))      # halfway, odd neighbour below
    flat[idx[5]] = np.float32(2 ** -130)               # subnormal
    return a


def _np_input(y):
    """y [D, S, S, C] fp32 (the joined map) -> V hi, lo [16, G, C]."""
    D, _, _, C = y.shape
    p = np.zeros((D, S + 2, S + 2, C), np.float32)
    p[:, 1:-1, 1:-1] = y
    d = [[p[:, i:i + S:2, j:j + S:2].reshape(D * NT * NT, C) for j in range(4)] for i in range(4)]
    w = [[None] * 4 for _ in range(4)]
    for j in range(4):
        w[0][j] = d[0][j] - d[2][j]
        w[1][j] = d[1][j] + d[2][j]
        w[2][j] = d[2][j] - d[1][j]
        w[3][j] = d[1][j] - d[3][j]
    v = []
    for i in range(4):
        v += [w[i][0] - w[i][2], w[i][1] + w[i][2], w[i][2] - w[i][1], w[i][1] - w[i][3]]
    return _split(np.stack(v))


def _np_output(m, D, bias, relu):
    """M [16, G, C] fp32 -> the layer output as (hi, lo) [D, S, S, C]."""
    q = m.reshape(4, 4, -1, m.shape[-1])
    s0 = [(q[0, j] + q[1, j]) + q[2, j] for j in range(4)]
    s1 = [(q[1, j] - q[2, j]) - q[3, j] for j in range(4)]
    out = np.zeros((D, NT, NT, 2, 2, m.shape[-1]), np.float32)
    for i, s in enumerate((s0, s1)):
        for k in range(2):
            o = ((s[0] + s[1]) + s[2]) if k == 0 else ((s[1] - s[2]) - s[3])
            o = o + bias
            if relu:
                o = np.where(o > 0, o, np.float32(0))
            out[:, :, :, i, k] = o.reshape(D, NT, NT, -1)
    hi, lo = _split(out.transpose(0, 1, 3, 2, 4, 5).reshape(D, S, S, -1))
    return hi, lo


def _same_bits(a, b):
    return np.array_equal(np.ascontiguousarray(a, np.float32).view(np.uint32), np.ascontiguousarray(b, np.float32).view(np.uint32))


@pytest.mark.parametrize('D,C', [(832, 64), (37, 512)])
def test_wino_input_bit_exact(D, C):
    rng = np.random.RandomState(D)
    hi, lo = _split(_edge_values(rng, (D, S, S, C)))
    x = _np_to_pairs(hi, lo)
    v = torch.empty((16, D * NT * NT, 2 * C), dtype=torch.bfloat16, device='cuda')
    cv.wino_input(x, v)
    vh, vl = _pairs_to_np(v)
    rh, rl = _np_input(hi + lo)
    assert _same_bits(vh, rh) and _same_bits(vl, rl)


@pytest.mark.parametrize('D,C', [(832, 64), (37, 512)])
def test_wino_output_transforms_bit_exact(D, C):
    rng = np.random.RandomState(D + 1)
    G = D * NT * NT
    m = _edge_values(rng, (16, G, C))
    bias = rng.randn(C).astype(np.float32)
    mt = torch.from_numpy(m).cuda()
    bt = torch.from_numpy(bias).cuda()
    y = torch.empty((D, 1, S, S, 2 * C), dtype=torch.bfloat16, device='cuda')
    cv.wino_output(mt, D, S, C, bt, True, y)
    yh, yl = _pairs_to_np(y)
    rh, rl = _np_output(m, D, bias, True)
    assert _same_bits(yh.reshape(rh.shape), rh) and _same_bits(yl.reshape(rl.shape), rl)
    # fused: exactly the output transform followed by the input transform of the joined pairs
    v = torch.empty((16, G, 2 * C), dtype=torch.bfloat16, device='cuda')
    cv.wino_output_input(mt, D, S, C, bt, True, v)
    vh, vl = _pairs_to_np(v)
    qh, ql = _np_input(rh + rl)
    assert _same_bits(vh, qh) and _same_bits(vl, ql)
    # no bias, no ReLU
    cv.wino_output(mt, D, S, C, None, False, y)
    yh, yl = _pairs_to_np(y)
    rh, rl = _np_output(m, D, np.zeros(C, np.float32), False)
    assert _same_bits(yh.reshape(rh.shape), rh) and _same_bits(yl.reshape(rl.shape), rl)


def _rand_pairs(shape, scale, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return cv.split_bf16(torch.randn(shape, device='cuda', generator=g) * scale)


@pytest.mark.parametrize('cin', [256, 512])
def test_wino_gemm_vs_fp64(cin):
    """M_xi = V_xi U_xi^T at D = 104 (G = 5096: 2560 tiles, > 19 per CTA).  The kernel forms hi*hi + lo*hi + hi*lo of
    exact bf16 operands (products exact in fp32) and drops lo*lo, at most 2^-18 |V||U| per term; its 3 Cin fp32
    accumulations add at most 2^-22 (the tensor cores truncate) of the running sum each, bounded by sum |V||U|."""
    D, cout = 104, 512
    G = D * NT * NT
    v = _rand_pairs((16, G, cin), 1.0, 1)
    u = _rand_pairs((16, cout, cin), 0.05, 2)
    m = torch.empty((16, G, cout), dtype=torch.float32, device='cuda')
    o = cv.wino_plan(G, cin, cout)
    assert o.tiles >= 3 * 132
    cv.wino_gemm(v, u, m, G)
    vf, uf = cv.join_split(v).double(), cv.join_split(u).double()
    ref = torch.bmm(vf, uf.transpose(1, 2))
    a = torch.bmm(vf.abs(), uf.abs().transpose(1, 2))
    bound = a * (2.0 ** -17 + 3 * cin * 2.0 ** -22)
    err = (m.double() - ref).abs()
    assert bool((err <= bound).all()), (err / a.clamp_min(1e-30)).max().item()


@pytest.mark.parametrize('D', [1, 37, 104, 832])
@pytest.mark.parametrize('cin', [256, 512])
def test_wino_gemm_exact_on_integer_pairs(cin, D):
    """M_xi = sum_c Vh Uh + Vl Uh + Vh Ul exactly, on independent integer hi / lo halves of V and U (the exact forward
    check of test_conv_reference: every partial sum is an fp32 value while 3 a^2 Cin < 2^22), so a dropped, repeated or
    misaddressed (k-block, product) shows.  D = 832 is the benchmarked 8 clips x 104 keypoint slots (G = 40768)."""
    from test_conv_reference import EXACT_LIMIT, exact_bound, int_amplitude
    cout = 512
    G = D * NT * NT
    a = int_amplitude(cin)
    assert exact_bound(a, cin, True, 1.0, 0.0) < EXACT_LIMIT
    g = torch.Generator(device='cuda').manual_seed(cin * 1000 + D)

    def ints(shape):
        return torch.randint(-a, a + 1, shape, generator=g, device='cuda').double()
    vh, vl, uh, ul = ints((16, G, cin)), ints((16, G, cin)), ints((16, cout, cin)), ints((16, cout, cin))
    v = torch.cat([vh, vl], -1).to(torch.bfloat16).contiguous()
    u = torch.cat([uh, ul], -1).to(torch.bfloat16).contiguous()
    m = torch.full((16, G, cout), float('nan'), dtype=torch.float32, device='cuda')
    cv.wino_gemm(v, u, m, G)
    terms = {'V_hi*U_hi': (vh, uh), 'V_lo*U_hi': (vl, uh), 'V_hi*U_lo': (vh, ul)}
    ref = sum(torch.bmm(p, q.transpose(1, 2)) for p, q in terms.values())
    assert float((torch.bmm(vl, ul.transpose(1, 2)) != 0).double().mean()) > 0.5      # lo*lo added would show
    bad = m.double() != ref
    if bool(bad.any()):
        xi, gi, co = [int(i) for i in torch.unravel_index(bad.view(-1).nonzero()[0, 0], bad.shape)]
        diff = float(m[xi, gi, co]) - float(ref[xi, gi, co])
        hits = ['%s of k-block %d %s' % (n, kb, 'dropped' if c == -diff else 'added twice')
                for n, (p, q) in terms.items() for kb in range(cin // 64)
                for c in [float((p[xi, gi, kb * 64:(kb + 1) * 64] * q[xi, co, kb * 64:(kb + 1) * 64]).sum())]
                if c != 0 and abs(c) == abs(diff)]
        pytest.fail('%d wrong entries of M; first (component %d, tile %d, Cout %d): difference %r; equals a single term: %s'
                    % (int(bad.sum()), xi, gi, co, diff, '; '.join(hits) or 'none'))


def _layer_inputs(D, cin, cout, seed):
    rng = np.random.RandomState(seed)
    xs = np.abs(rng.randn(D, 1, S, S, cin)).astype(np.float32)         # post-ReLU activations
    hi, lo = _split(xs)
    w = (rng.randn(cout, cin, 3, 3) / np.sqrt(9 * cin)).astype(np.float32)
    b = (0.1 * rng.randn(cout)).astype(np.float32)
    return hi, lo, w, b


@pytest.mark.parametrize('cin', [256, 512])
def test_wino_layer_vs_fp64_direct_conv(cin):
    """One head layer (input transform, GEMM, output transform with bias and ReLU) against the fp64 3x3 conv of the
    values the kernels read (x = hi + lo, the fp32 filter), within STEP_TOL['bf16x3'] = 1e-4 max|ref|."""
    import torch.nn.functional as F
    D, cout = 104, 512
    hi, lo, w, b = _layer_inputs(D, cin, cout, cin)
    x = _np_to_pairs(hi, lo).view(D, 1, S, S, 2 * cin)
    G = D * NT * NT
    v = torch.empty((16, G, 2 * cin), dtype=torch.bfloat16, device='cuda')
    m = torch.empty((16, G, cout), dtype=torch.float32, device='cuda')
    y = torch.empty((D, 1, S, S, 2 * cout), dtype=torch.bfloat16, device='cuda')
    bt = torch.from_numpy(b).cuda()
    cv.wino_input(x, v)
    cv.wino_gemm(v, cv.pack_wino_weight(w), m, G)
    cv.wino_output(m, D, S, cout, bt, True, y)
    xd = torch.from_numpy((hi.astype(np.float64) + lo)[:, 0]).cuda().permute(0, 3, 1, 2)
    ref = F.relu(F.conv2d(xd, torch.from_numpy(w).double().cuda(), torch.from_numpy(b).double().cuda(), padding=1))
    ref = ref.permute(0, 2, 3, 1)
    got = cv.join_split(y)[:, 0].double()
    tol = 1e-4 * ref.abs().max().item()
    err = (got - ref).abs().max().item()
    direct = cv.conv3d(x, cv.pack_weight(torch.from_numpy(w), cv.BF16X3), (1, 3, 3), pad=(0, 1, 1), bias=bt, relu=True,
                       dtype=cv.BF16X3)
    err_direct = (cv.join_split(direct)[:, 0].double() - ref).abs().max().item()
    assert err <= tol, (err, tol, err_direct)


def test_wino_head_vs_direct_head():
    """Eight 3x3 convs (256 -> 512, then 512 -> 512) and the sub-pixel deconv, Winograd against direct, on the same
    RoI features; the deconv's fp32 low-res maps agree within 5e-4 max|direct| (the teacher-forced heat-map bound of
    the engine tests)."""
    from detectandtrack_b200.modeling.engine import DetectionEngine, _Conv
    D = 104
    rng = np.random.RandomState(7)
    convs = []
    cin = 256
    for i in range(8):
        w = (rng.randn(512, cin, 3, 3) * np.sqrt(2.0 / (9 * cin))).astype(np.float32)
        c = _Conv(torch, w, cv.BF16X3, None, (0.01 * rng.randn(512)).astype(np.float32), pad=(0, 1, 1), relu=True)
        c.wu = cv.pack_wino_weight(w)
        convs.append(c)
        cin = 512
    deconv = _Conv(torch, (0.01 * rng.randn(68, 512, 3, 3)).astype(np.float32), cv.BF16X3, None, np.zeros(68, np.float32),
                   pad=(0, 1, 1))
    hi, lo = _split(np.abs(rng.randn(D, 1, S, S, 256)).astype(np.float32))
    x = _np_to_pairs(hi, lo).view(D, 1, S, S, 512)
    eng = types.SimpleNamespace(torch=torch, _geom={}, kps_convs=convs)
    yw = DetectionEngine._kps_convs_wino(eng, x)
    yd = x
    for c in convs:
        yd = c(yd)
    lw = torch.empty((D, 1, S, S, 68), dtype=torch.float32, device='cuda')
    ld = torch.empty_like(lw)
    deconv(yw, out_f32=True, out=lw)
    deconv(yd, out_f32=True, out=ld)
    err = (lw - ld).abs().max().item()
    assert err <= 5e-4 * ld.abs().max().item(), (err, ld.abs().max().item())
    assert (cv.join_split(yw) - cv.join_split(yd)).abs().max().item() <= 1e-3 * cv.join_split(yd).abs().max().item()


@pytest.mark.parametrize('wl,mode,taken', [('r50fpn3d', 'bf16x3', True), ('r50fpn3d', 'bf16x3h', True),
                                           ('r50fpn3d', 'tf32x3', False), ('r18tube', 'bf16x3', False)])
def test_engine_takes_the_winograd_path(wl, mode, taken):
    import step_launches as sl
    rec = sl.record((wl, mode))
    names = [name for name, a, _ in rec.calls
             if name.startswith('dt_wino') or (name == 'dt_conv3d' and a[0]._obj.Hi == S and a[0]._obj.kH == 3)]
    n = rec.facts['kps_convs']
    assert rec.facts['wino_kps'] == taken
    if taken:
        assert n == 8
        # then the sub-pixel deconv, the one direct 3x3 conv left on the 14 x 14 maps
        assert names == ['dt_wino_input'] + ['dt_wino_gemm', 'dt_wino_output_input'] * (n - 1) + \
            ['dt_wino_gemm', 'dt_wino_output', 'dt_conv3d'], names
    else:
        assert not any(x.startswith('dt_wino') for x in names), names
