"""Device-tensor API over csrc/conv_tc.cu (wgmma implicit-GEMM Conv3d/Conv2d/FC).
Tensors are NDHWC ([N, T, H, W, C], channels innermost); torch is only the memory
container.  See include/dt_b200.h (dt_conv_desc / dt_conv3d) for the contract."""
import ctypes as C

from .. import _lib as L

BF16, TF32 = 0, 1
TF32X3 = 2      # host-level mode: DT_DTYPE_TF32 kernels on [hi | lo] tf32 pairs (3 MMAs per k-block, ~fp32 accuracy)
BF16X3 = 3      # host-level mode: DT_DTYPE_BF16 kernels on [hi | lo] bf16 pairs (3 MMAs per k-block at the full
                # kind::f16 rate, 16 mantissa bits: the headline parity mode)
F16 = 4         # per-layer operand type, not an engine mode: fp16 x and w (DT_DTYPE_F16), one MMA per product at 11-bit
                # operands; used by the 'bf16x3h' engine mode for the post-hoc FPN convs
SPLIT_MODES = (TF32X3, BF16X3)
MODE_NAMES = {'bf16': BF16, 'tf32': TF32, 'tf32x3': TF32X3, 'bf16x3': BF16X3, 'bf16x3h': BF16X3}


def _dt(dtype, torch):
    return torch.float16 if dtype == F16 else (torch.bfloat16 if dtype in (BF16, BF16X3) else torch.float32)


def kernel_dtype(dtype):
    """Host-level mode -> DT_DTYPE_* of the kernels."""
    return 2 if dtype == F16 else (BF16 if dtype in (BF16, BF16X3) else TF32)


def pack_weight(w, dtype=BF16):
    """Caffe2 / torch filter (Cout, Cin, kT, kH, kW) [or 4-D (Cout, Cin, kH, kW), or 2-D FC
    (Cout, Cin)] -> tap-major [kT*kH*kW, Cout, Cin_pad] in the compute dtype; Cin is padded with
    zeros to a 16-byte multiple (TMA global-stride rule)."""
    torch = L.require_cuda()
    if w.dim() == 2:
        w = w[:, :, None, None, None]
    elif w.dim() == 4:
        w = w[:, :, None, :, :]
    Cout, Cin, kT, kH, kW = w.shape
    mult = 8 if dtype in (BF16, BF16X3, F16) else 4
    Cp = (Cin + mult - 1) // mult * mult
    out = torch.zeros((kT * kH * kW, Cout, Cp), dtype=torch.bfloat16 if dtype == BF16 else (torch.float16 if dtype == F16 else torch.float32), device='cuda')
    out[:, :, :Cin] = w.to('cuda').permute(2, 3, 4, 0, 1).reshape(kT * kH * kW, Cout, Cin).to(out.dtype)
    if dtype == TF32:
        out = round_tf32(out)
    elif dtype == TF32X3:
        out = split_tf32(out)                         # [taps, Cout, 2*Cp] = [hi | lo]
    elif dtype == BF16X3:
        out = split_bf16(out)                         # [taps, Cout, 2*Cp] bf16 = [hi | lo]
    return out


def split_bf16(t):
    """fp32 [..., C] -> bf16 [..., 2C] = [hi | lo], hi = bf16(t), lo = bf16(t - hi) (bf16x3 storage)."""
    torch = L.require_cuda()
    hi = t.to(torch.bfloat16)
    lo = (t - hi.float()).to(torch.bfloat16)
    return torch.cat([hi, lo], dim=-1).contiguous()


def split_for(dtype, t):
    """fp32 tensor -> the split storage of `dtype` (TF32X3: fp32 tf32 pairs, BF16X3: bf16 pairs)."""
    return split_bf16(t.float()) if dtype == BF16X3 else split_tf32(t.float())


def join_split(t):
    """[..., 2C] split rows (either storage type) -> fp32 values hi + lo."""
    c = t.shape[-1] // 2
    return t[..., :c].float() + t[..., c:].float()


def split_tf32(t):
    """fp32 [..., C] -> [..., 2C] = [hi | lo] with hi = tf32(t), lo = tf32(t - hi) (3xTF32 storage)."""
    torch = L.require_cuda()
    hi = round_tf32(t)
    lo = round_tf32(t - hi)
    return torch.cat([hi, lo], dim=-1).contiguous()


def join_tf32(t):
    """Inverse of split_tf32 (exact: hi + lo fits fp32)."""
    c = t.shape[-1] // 2
    return t[..., :c] + t[..., c:]


def round_tf32(t):
    """Round an fp32 tensor to the nearest (even) tf32-representable value.  The tf32 MMA
    ignores the low 13 mantissa bits of its operands; feeding it pre-rounded values makes the
    truncation exact instead of a one-sided error."""
    torch = L.require_cuda()
    u = t.contiguous().view(torch.int32)
    u = u + 0xFFF + ((u >> 13) & 1)
    return (u & ~0x1FFF).view(torch.float32)


def conv3d(x, w_packed, ksize, stride=(1, 1, 1), pad=(0, 0, 0), scale=None, bias=None,
           residual=None, res_mode=0, relu=False, out_f32=None, dtype=BF16, cin=None, out=None, round_tf32=None,
           split_out=None, time_major=False, out_frames=None):
    """x [N,T,H,W,Cx] (first `cin` channels are the conv input); returns y [N,To,Ho,Wo,Cout].
    time_major: y is stored [To,N,Ho,Wo,Cout] and returned as the permuted [N,To,...] view, so y[:, t:t+1]
    is contiguous (the centre-frame link needs no copy).
    out_frames=(first, count): compute only those output frames (y has `count` frames)."""
    torch = L.require_cuda()
    assert x.is_cuda and x.dim() == 5 and x.is_contiguous()
    assert x.dtype == _dt(dtype, torch), (x.dtype, dtype)
    N, Ti, Hi, Wi, Cx = x.shape
    taps, Cout, w_ld = w_packed.shape
    kT, kH, kW = ksize
    assert taps == kT * kH * kW
    x3 = dtype in SPLIT_MODES
    if x3:
        cin = cin if cin is not None else min(Cx // 2, w_ld // 2)
        if split_out is None:
            split_out = out is None                  # intermediate activations stay split; given buffers are final
        if out_f32 is None:
            out_f32 = (dtype == TF32X3) or not split_out
        assert out_f32 == (dtype == TF32X3) or not split_out, 'split outputs are fp32 pairs (tf32x3) / bf16 pairs (bf16x3)'
    else:
        split_out = bool(split_out) and dtype == F16       # an fp16-operand conv may write bf16 pairs for a bf16x3 consumer
    cin = cin if cin is not None else min(Cx, w_ld)
    sT, sH, sW = stride
    pT, pH, pW = pad
    To = (Ti + 2 * pT - kT) // sT + 1
    Ho = (Hi + 2 * pH - kH) // sH + 1
    Wo = (Wi + 2 * pW - kW) // sW + 1
    t_first, t_count = (0, 0) if out_frames is None else (int(out_frames[0]), int(out_frames[1]))
    if t_count:
        assert 0 <= t_first and t_first + t_count <= To and residual is None
        To = t_count
    if out_f32 is None:
        out_f32 = dtype == TF32
    if round_tf32 is None:
        round_tf32 = bool(out_f32) and dtype == TF32 and out is None      # intermediate activations
    if x3:
        round_tf32 = False
    odt = torch.float32 if out_f32 else torch.bfloat16
    if out is None:
        cw = 2 * Cout if split_out else Cout
        out = torch.empty((To, N, Ho, Wo, cw) if time_major else (N, To, Ho, Wo, cw), dtype=odt, device='cuda')
    else:
        assert not time_major, 'time_major allocates its own output'
    assert out.dtype == odt and out.is_contiguous()
    d = L.ConvDesc(N=N, Ti=Ti, Hi=Hi, Wi=Wi, Cin=cin, Cout=Cout, kT=kT, kH=kH, kW=kW, sT=sT, sH=sH, sW=sW,
                   pT=pT, pH=pH, pW=pW, in_ld=Cx, w_ld=w_ld, out_ld=out.shape[-1],
                   res_ld=(residual.shape[-1] if residual is not None else 0), dtype=kernel_dtype(dtype),
                   out_f32=int(out_f32), relu=int(relu), res_mode=int(res_mode),
                   x3=(1 if x3 else 0) | (2 if split_out else 0), in_lo_off=0, out_lo_off=0, res_lo_off=0,
                   out_round_tf32=int(bool(round_tf32)), out_time_major=int(bool(time_major)), out_t_first=t_first,
                   out_t_count=t_count)
    if residual is not None:
        assert residual.dtype == odt and residual.is_contiguous()
    if scale is not None:
        assert scale.dtype == torch.float32 and scale.numel() == Cout
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.numel() == Cout
    L.call('dt_conv3d', C.byref(d), L.ptr(x), L.ptr(w_packed), L.ptr(scale), L.ptr(bias), L.ptr(residual),
           L.ptr(out), L.stream_ptr())
    return out.permute(1, 0, 2, 3, 4) if time_major else out


def pack_conv1_weight(w, dtype=BF16):
    """conv1 filter (Cout, 3, [1,] 7, 7) -> [7 (kh)][Cout][8 pixels x Cp] with element kw*Cp + c
    (dt_conv1_7x7s2); Cp = 8 (bf16) / 4 (tf32) channels per 16-byte pixel, zeros elsewhere."""
    torch = L.require_cuda()
    if w.dim() == 5:
        w = w[:, :, 0]
    Cout, Cin, kh, kw = w.shape
    assert (kh, kw) == (7, 7) and Cin <= 3 + 1
    Cp = 4 if dtype == TF32 else 8
    wk = w.to('cuda').float().permute(2, 0, 3, 1)                                  # (kh, Cout, kw, c)
    if dtype == BF16X3:
        # split-pixel blob [hi3 | lo3 | 0 0]: block 2*kh = [W_hi | W_hi] (x_hi*W_hi + x_lo*W_hi in one MMA),
        # block 2*kh + 1 = [W_lo | 0] (x_hi*W_lo)
        assert Cin == 3
        hi = wk.to(torch.bfloat16)
        lo = (wk - hi.float()).to(torch.bfloat16)
        out = torch.zeros((7, 2, Cout, 8, 8), dtype=torch.bfloat16, device='cuda')
        out[:, 0, :, :7, 0:3] = hi
        out[:, 0, :, :7, 3:6] = hi
        out[:, 1, :, :7, 0:3] = lo
        return out.reshape(14, Cout, 64)
    out = torch.zeros((7, Cout, 8, Cp), dtype=_dt(dtype, torch), device='cuda')
    out[:, :, :7, :Cin] = wk.to(out.dtype)
    out = out.reshape(7, Cout, 8 * Cp)
    return round_tf32(out) if dtype == TF32 else out


def conv1_7x7s2(x_padded, w_packed, hw, scale=None, bias=None, relu=True, dtype=BF16, out_f32=None):
    """x_padded [F, 2, (Hp+6)/2, Wp+8, Cp] (dense_ops.prep_clip(border=(3, 4), row_planes=True)) -> [F, Hp/2, Wp/2, Cout]."""
    torch = L.require_cuda()
    F, two, Hh, Wt, Cp = x_padded.shape
    Hp, Wp = hw
    assert two == 2 and 2 * Hh == Hp + 6 and Wt == Wp + 8 and x_padded.is_contiguous()
    Cout = w_packed.shape[1]
    x3 = dtype == BF16X3                       # split-pixel blob, 14 weight blocks, [hi | lo] bf16 pair output
    if out_f32 is None:
        out_f32 = dtype == TF32
    assert not (x3 and out_f32)
    ld = 2 * Cout if x3 else Cout
    y = torch.empty((F, Hp // 2, Wp // 2, ld), dtype=torch.float32 if out_f32 else torch.bfloat16, device='cuda')
    L.call('dt_conv1_7x7s2', L.ptr(x_padded), F, Hp, Wp, Cp, L.ptr(w_packed), Cout, L.ptr(scale), L.ptr(bias), int(relu),
           kernel_dtype(dtype), int(out_f32), int(bool(out_f32) and dtype == TF32), int(x3), L.ptr(y), ld, L.stream_ptr())
    return y


def conv1_7x7s2_f32(blob, w, scale, bias, out_bf16=False):
    """Split-storage modes' conv1: exact fp32 (dt_conv1_7x7s2_f32).  blob [F, Hp, Wp, Cp] raw fp32;
    w (64, 3, [1,] 7, 7) -> [F, Hp/2, Wp/2, 128] as [hi | lo] (tf32 pairs in fp32, or bf16 pairs)."""
    torch = L.require_cuda()
    F, Hp, Wp, Cp = blob.shape
    y = torch.empty((F, Hp // 2, Wp // 2, 128), dtype=torch.bfloat16 if out_bf16 else torch.float32, device='cuda')
    L.call('dt_conv1_7x7s2_f32', L.ptr(blob), F, Hp, Wp, Cp, L.ptr(w), L.ptr(scale), L.ptr(bias), int(bool(out_bf16)),
           L.ptr(y), L.stream_ptr())
    return y


def pack_conv1_weight_f32(w):
    """(64, 3, [1,] 7, 7) -> [7][7][3][64] fp32 for dt_conv1_7x7s2_f32."""
    torch = L.require_cuda()
    if w.dim() == 5:
        w = w[:, :, 0]
    assert tuple(w.shape) == (64, 3, 7, 7)
    return w.to('cuda').float().permute(2, 3, 1, 0).contiguous()
