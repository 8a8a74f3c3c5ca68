"""CPU: the Winograd F(2x2, 3x3) keypoint-head pieces that run without a GPU — the filter transform U = G g G^T, the plan
dt_wino_gemm launches, and the host-side argument checks of the dt_wino_* entry points."""
import ctypes as C

import numpy as np
import pytest

from detectandtrack_b200 import _lib as L
from detectandtrack_b200.ops import conv as cv


def test_wino_filter_is_G_g_Gt():
    rng = np.random.RandomState(0)
    w = rng.randn(6, 5, 3, 3).astype(np.float32)
    G = np.array([[1, 0, 0], [.5, .5, .5], [.5, -.5, .5], [0, 0, 1]], np.float64)
    u = cv.wino_filter(w)
    assert u.shape == (16, 6, 5) and u.dtype == np.float32
    for o in range(6):
        for c in range(5):
            ref = (G @ w[o, c].astype(np.float64) @ G.T).astype(np.float32)
            assert np.array_equal(u[:, o, c].reshape(4, 4), ref)
    assert np.array_equal(cv.wino_filter(w[:, :, None]), u)          # 5-D filter with kT = 1


def test_wino_filter_reproduces_the_direct_conv_in_fp64():
    """Y = A^T [U . V] A over the 4 x 4 patch equals the 3x3 correlation of its 2 x 2 outputs (the layout the kernels
    assume: component xi = 4 i + j, rows first)."""
    rng = np.random.RandomState(1)
    g = rng.randn(1, 1, 3, 3)
    d = rng.randn(4, 4)
    U = cv.wino_filter(g).astype(np.float64).reshape(4, 4)
    Bt = np.array([[1, 0, -1, 0], [0, 1, 1, 0], [0, -1, 1, 0], [0, 1, 0, -1]], np.float64)
    At = np.array([[1, 1, 1, 0], [0, 1, -1, -1]], np.float64)
    y = At @ (U * (Bt @ d @ Bt.T)) @ At.T
    ref = np.array([[(d[r:r + 3, c:c + 3] * g[0, 0]).sum() for c in range(2)] for r in range(2)])
    assert np.abs(y - ref).max() < 1e-6


@pytest.mark.parametrize('D,cin', [(104, 256), (104, 512), (832, 512), (37, 512)])
def test_wino_gemm_plan(D, cin):
    G = D * 49
    o = cv.wino_plan(G, cin, 512)
    assert (o.BN, o.TH, o.TW, o.TT, o.TB) == (128, 1, 128, 1, 1)       # one component per M tile
    assert o.kiters == 3 * cin // 64
    assert o.tiles == 16 * (-(-G // 128)) * 4
    assert o.stages >= 2 and o.smem_bytes <= 227 * 1024
    # the same operand ring / staging as the pointwise bf16x3 conv of that K and N (the conv planner's split)
    d = L.ConvDesc(N=16, Ti=1, Hi=1, Wi=G, Cin=cin, Cout=512, kT=1, kH=1, kW=1, sT=1, sH=1, sW=1, in_ld=2 * cin,
                   w_ld=2 * cin, out_ld=512, dtype=0, out_f32=1, x3=1)
    p = L.ConvPlan()
    assert L.lib().dt_conv_plan(C.byref(d), 0, C.byref(p)) == 0
    assert (o.stages, o.ks, o.ncbuf, o.nrbuf, o.smem_bytes, o.stage_bytes) == \
        (p.stages, p.ks, p.ncbuf, p.nrbuf, p.smem_bytes, p.stage_bytes)


def _cases():
    return [
        ('dt_wino_gemm', (None, None, None, 0, 512, 512, None), b'G=0'),
        ('dt_wino_gemm', (None, None, None, 49, 100, 512, None), b'Cin=100'),
        ('dt_wino_gemm', (None, None, None, 49, 512, 512, None), b'null tensor'),
        ('dt_wino_plan', (49, 512, 96, None), b'null pointer'),
        ('dt_wino_input', (None, 4, 13, 64, None, None), b'S=13'),
        ('dt_wino_input', (None, 4, 14, 64, None, None), b'null'),
        ('dt_wino_output_input', (None, 4, 14, 96, None, 1, None, None), b'C=96'),
        ('dt_wino_output_input', (None, 0, 14, 64, None, 1, None, None), b'D=0'),
        ('dt_wino_output', (None, 4, 18, 64, None, 1, None, None), b'S=18'),
        ('dt_wino_output', (None, 4, 14, 64, None, 1, None, None), b'null'),
    ]


@pytest.mark.parametrize('name,args,msg', _cases(), ids=['%s-%d' % (c[0], i) for i, c in enumerate(_cases())])
def test_wino_entry_points_reject_bad_arguments_without_a_gpu(name, args, msg):
    lib = L.lib()
    rc = getattr(lib, name)(*args)
    assert rc != 0, name
    assert msg in lib.dt_last_error(), (name, lib.dt_last_error())
    with pytest.raises(RuntimeError, match=name):
        L.check(rc, name)


def test_wino_plan_rejects_a_bad_shape():
    o = L.ConvPlan()
    assert L.lib().dt_wino_plan(49, 512, 96, C.byref(o)) != 0
    assert b'Cout=96' in L.lib().dt_last_error()
