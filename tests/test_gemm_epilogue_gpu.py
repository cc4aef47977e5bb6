"""The epilogues of the wgmma GEMM / conv kernels (gemm_tc.cu: gemm_tc_kernel<64|128|256>, conv_halo_kernel<64|128>)
and of the RGB stem (rgb_conv.cu), element by element against fp64, one pinned launch path per case.

Each case names one call of ops.linear / ops.conv / ops.conv_up2x / ops.conv_rgb: the shape; the epilogue (activation,
residual dtype, SFT and its weight, ReLU after the residual, output dtype and layout, fused GroupNorm statistics); the
views it passes (output offset and row-pitch padding, input channel slice, residual / scale pitch and offset, bias
offset, output aliasing the residual); and the launch it must take, as the library's launch profiler describes it:
kernel, BN, mode, tile t{frames}x{rows}x{columns}, e (1: TMA-store epilogue, 0: direct per-thread stores) and r (halo
kernel: weights resident).  A dispatch change that moves a case off its path fails that case, and
test_cases_cover_the_required_paths keeps the matrix covering the paths written out in REQUIRED.

Inputs.  Weights carry a per-output-channel scale spread over 2^-6 .. 2^6 and activations a per-pixel (per-row)
scale over 2^-2 .. 2^2; bias, residual and the SFT residual are scaled per channel like the weights.  So an error
confined to a small channel, or to some pixels, is not hidden under the largest values.

Bound.  The reference is fp64 on the bf16-rounded operands the kernel reads.  Every written element must satisfy
    |got - ref| <= u_out |ref| + eps S,
where S is the element's own magnitude sum: Sa = sum_k |a_k w_k| + |b|, times the largest slope of the activation
(1.2 covers GELU's 1.13 and SiLU's 1.10) plus |act(z)| for the activations computed with ex2 / rcp approximations
(their error is relative to their result), plus |residual|; for SFT, y = r + w (r s + z): |w| Sa + |r| + |w| |r s|.
u_out is 2^-8 for bf16 outputs (the rounding is 2^-9; the rest is slack for rounding a value already off by eps S) and
0 for fp32.  eps covers the fp32 accumulation and the activation approximations; EPS is set per kernel family from the
worst err / S measured over this matrix (printed at the end of the module), see its comment.

Poison.  Every byte a call must not write (row padding of the output view, the elements before its offset, the rows
after it) and every byte it must not read (input channels [Cin, ldx), A / W columns [K, ld), residual and scale
padding, bias padding, weight rows past Cout) is NaN; outputs are NaN before the call.  Afterwards the output view must
be finite and within the bound, and every other element of its buffer bit-identical to what it was.

Identity.  The same plain epilogue (act none / relu / lrelu, no FMA that could contract differently) gives the same
bits on the TMA-store path and on the direct path; a linear launched as 64-column slices (BN = 64) gives the same bits
as one BN = 128 launch: every output element accumulates its k-blocks in the same order in both."""
import csv
import math
import os
import re

import pytest
import torch
import torch.nn.functional as F

DEV = 'cuda'
gpu = pytest.mark.gpu

U_BF16 = 2.0 ** -8
# Worst err / S over this matrix, measured on an H100 80GB HBM3 (700 W): linear 2^-22.0, conv 2^-20.6, halo3 2^-21.4;
# rgb_conv writes bf16 only, and no element of it exceeded the rounding term.  eps is the next power of two with at
# least a factor 2 of margin, the rgb stem's that of the linear (its k loop is at most 160 products long).
EPS = {'linear': 2.0 ** -20, 'conv': 2.0 ** -19, 'halo3': 2.0 ** -20, 'rgb_conv': 2.0 ** -20}
WORST = {}

ACT_CODE = {'none': 0, 'gelu': 1, 'silu': 2, 'lrelu': 3, 'relu': 4, 'sigmoid': 5}
SMOOTH = ('gelu', 'silu', 'sigmoid')


def _act(z, act):
    if act == 'gelu':
        return F.gelu(z)
    if act == 'silu':
        return F.silu(z)
    if act == 'lrelu':
        return F.leaky_relu(z, 0.2)
    if act == 'relu':
        return F.relu(z)
    if act == 'sigmoid':
        return torch.sigmoid(z)
    return z


# ------------------------------------------------------------------------------------------------ the case matrix
_DEFAULTS = dict(F=1, H=0, W=0, Cin=0, N=0, M=0, K=0, ksize=3, stride=1, pad_lo=1, act='none', bias=True, boff=0,
                 res=None, rpad=0, roff=0, sft=None, apad=0, aoff=0, rar=False, out='bf16', gn=False, ooff=0, opad=0,
                 xpad=0, kpad=0, alias=False, wide=False)


def case(entry, launch, **kw):
    c = dict(_DEFAULTS)
    for k in kw:
        assert k in c, k
    c.update(kw, entry=entry, launch=launch)
    return c


def case_id(c):
    if c['entry'] == 'linear':
        s = 'lin-M%s-N%d-K%d' % ('wide' if c['wide'] else c['M'], c['N'], c['K'])
    elif c['entry'] == 'rgb':
        s = 'rgb-%dx%d-k%ds%d-N%d' % (c['H'], c['W'], c['ksize'], c['stride'], c['N'])
    else:
        s = '%s-F%s-%dx%d-Cin%d-N%d' % (c['entry'], 'wide' if c['wide'] else c['F'], c['H'], c['W'], c['Cin'], c['N'])
        if c['entry'] == 'conv':
            s += '-k%ds%dp%d' % (c['ksize'], c['stride'], c['pad_lo'])
    s += '-' + c['act'] + '-' + c['out']
    for k in ('res', 'sft'):
        if c[k] is not None:
            s += '-%s%s' % (k, c[k])
    for k in ('rar', 'gn', 'alias'):
        if c[k]:
            s += '-' + k
    for k in ('boff', 'rpad', 'roff', 'apad', 'aoff', 'ooff', 'opad', 'xpad', 'kpad'):
        if c[k]:
            s += '-%s%d' % (k, c[k])
    return s


L, C, U, R = 'linear', 'conv', 'up2x', 'rgb'
CASES = [
    # ---------------- linear: every activation, the ARM / FFM sigmoid shapes (a few rows x 128 / 256)
    *[case(L, 'linear BN128 e1', M=300, N=256, K=192, act=a) for a in ACT_CODE],
    case(L, 'linear BN128 e1', M=3, N=128, K=256, act='sigmoid'),
    case(L, 'linear BN128 e1', M=8, N=256, K=512, act='sigmoid', out='f32'),
    case(L, 'linear BN64 e1', M=5, N=64, K=128, act='sigmoid', out='f32'),
    # ---------------- linear tails: M in {1, 127, 129} x N in {3, 40, 200}, K % 64 != 0 with NaN past K
    *[case(L, lau, M=m, N=n, K=200, kpad=kp, act=a, out=o)
      for (m, n, kp, a, o, lau) in [
          (1, 3, 8, 'none', 'bf16', 'linear BN64 e0'), (1, 40, 24, 'gelu', 'f32', 'linear BN64 e1'),
          (1, 200, 56, 'relu', 'bf16', 'linear BN128 e1'), (127, 3, 8, 'silu', 'f32', 'linear BN64 e0'),
          (127, 40, 56, 'lrelu', 'bf16', 'linear BN64 e1'), (127, 200, 24, 'none', 'f32', 'linear BN128 e1'),
          (129, 3, 24, 'gelu', 'bf16', 'linear BN64 e0'), (129, 40, 8, 'none', 'f32', 'linear BN64 e1'),
          (129, 200, 8, 'silu', 'bf16', 'linear BN128 e1')]],
    case(L, 'linear BN128 e1', M=200, N=512, K=57, kpad=7, opad=32, ooff=512),
    # ---------------- linear on 256-wide tiles with a ragged last n-tile (N = 448) and a ragged last row tile
    case(L, 'linear BN256 e1', wide=True, N=448, K=576, act='gelu', res='bf16', kpad=64),
    case(L, 'linear BN256 e1', wide=True, N=448, K=576, res='f32', out='f32'),
    case(L, 'linear BN256 e0', wide=True, N=448, K=576, act='silu', res='f32'),
    # ---------------- linear epilogues: mixed residual dtypes, ReLU after the residual, padded / offset views
    case(L, 'linear BN128 e0', M=300, N=256, K=192, res='f32', act='gelu'),
    case(L, 'linear BN128 e0', M=300, N=256, K=192, res='bf16', out='f32', act='silu'),
    case(L, 'linear BN128 e0', M=300, N=256, K=192, res='bf16', out='f32', act='relu', rar=True),
    case(L, 'linear BN128 e1', M=300, N=256, K=192, res='bf16', act='relu', rar=True, rpad=16, opad=8),
    case(L, 'linear BN128 e0', M=300, N=256, K=192, res='bf16', rpad=3, roff=1, opad=4),
    case(L, 'linear BN64 e1', M=300, N=64, K=192, res='f32', out='f32', act='lrelu', alias=True),
    case(L, 'linear BN128 e1', M=512, N=256, K=192, gn=True),
    # the fixed cases: bf16 output view offset by one element with ldo % 8 == 0, bias view offset by one float
    case(L, 'linear BN128 e0', M=300, N=256, K=192, ooff=1, opad=8),
    case(L, 'linear BN64 e0', M=300, N=64, K=192, ooff=1, opad=8, act='relu', res='bf16'),
    case(L, 'linear BN128 e1', M=300, N=256, K=192, boff=1, act='gelu'),
    case(L, 'linear BN64 e0', M=300, N=64, K=192, boff=1, out='f32', opad=1),
    case(L, 'linear BN256 e1', wide=True, N=448, K=576, boff=1),

    # ---------------- SFT on gemm_tc_kernel<128> (Engine.sft_tail's shift.2 conv): Cout 256 / 512, +- statistics
    case(C, 'conv BN128 s1 t1x4x32 e1', F=2, H=32, W=32, Cin=64, N=256, sft=0.7, res='bf16'),
    case(C, 'conv BN128 s1 t1x4x32 e1', F=2, H=32, W=32, Cin=64, N=256, sft=0.7, res='bf16', gn=True),
    case(C, 'conv BN128 s1 t1x4x32 e1', F=2, H=32, W=32, Cin=128, N=512, sft=1.0, res='bf16'),
    case(C, 'conv BN128 s1 t1x4x32 e1', F=2, H=32, W=32, Cin=128, N=512, sft=1.0, res='bf16', gn=True),
    case(C, 'conv BN128 s1 t1x4x32 e1', F=2, H=24, W=40, Cin=64, N=256, sft=0.5, res='bf16'),
    case(C, 'conv BN128 s1 t1x4x32 e1', F=2, H=32, W=32, Cin=64, N=256, sft=0.7, res='bf16', rpad=64, apad=128),
    # ---------------- SFT on gemm_tc_kernel<64>: Cout 64, frames too small for the halo tile, F % tn != 0
    case(C, 'conv BN64 s1 t2x8x8 e1', F=3, H=8, W=8, Cin=64, N=64, sft=0.7, res='bf16'),
    case(C, 'conv BN64 s1 t8x4x4 e1', F=3, H=4, W=4, Cin=128, N=64, sft=0.6, res='bf16'),
    # ---------------- SFT on the direct path: fp32 out, misaligned scale view, and on the halo kernel
    case(C, 'conv BN128 s1 t1x4x32 e0', F=2, H=32, W=32, Cin=64, N=256, sft=0.7, res='bf16', out='f32'),
    case(C, 'conv BN128 s1 t1x4x32 e0', F=2, H=32, W=32, Cin=64, N=256, sft=0.7, res='bf16', aoff=1),
    case(C, 'conv BN64 s1 t2x8x8 e0', F=3, H=8, W=8, Cin=64, N=64, sft=0.7, res='bf16', aoff=3, apad=8),
    case(C, 'halo3 BN128 e0 r0', F=2, H=16, W=16, Cin=64, N=128, sft=0.7, res='bf16', out='f32'),
    case(C, 'halo3 BN64 e0 r1', F=2, H=16, W=16, Cin=64, N=64, sft=0.7, res='bf16', aoff=1),
    case(C, 'halo3 BN128 e1 r0', F=2, H=24, W=40, Cin=64, N=128, sft=0.7, res='bf16'),
    # ---------------- every activation on the non-halo conv (BN 128 and 64) and on the halo kernel (BN 64 and 128)
    *[case(C, 'conv BN128 s1 t1x8x16 e1', F=2, H=8, W=16, Cin=64, N=96, act=a) for a in ACT_CODE],
    *[case(C, 'conv BN64 s1 t2x8x8 e1', F=3, H=8, W=8, Cin=64, N=64, act=a, out='f32') for a in ('gelu', 'sigmoid')],
    *[case(C, 'halo3 BN64 e1 r1', F=2, H=16, W=16, Cin=64, N=64, act=a) for a in ACT_CODE],
    *[case(C, 'halo3 BN128 e1 r0', F=2, H=24, W=40, Cin=96, N=128, act=a, out='f32', xpad=8)
      for a in ('silu', 'sigmoid', 'lrelu')],
    # ---------------- mixed residual dtypes on the non-halo conv (direct path) and the halo kernel
    case(C, 'conv BN128 s1 t1x8x16 e0', F=2, H=8, W=16, Cin=64, N=96, res='f32', act='silu'),
    case(C, 'conv BN128 s1 t1x8x16 e0', F=2, H=8, W=16, Cin=64, N=96, res='bf16', out='f32', act='gelu'),
    case(C, 'conv BN128 s1 t1x4x32 e0', F=2, H=32, W=32, Cin=64, N=256, res='f32'),
    case(C, 'halo3 BN64 e0 r1', F=2, H=16, W=16, Cin=64, N=64, res='bf16', out='f32', act='lrelu'),
    # ---------------- ReLU after the residual: stride-2 conv (BasicBlock downsample), and on the direct path
    case(C, 'conv BN128 s2 t1x8x16 e1', F=2, H=32, W=32, Cin=64, N=128, stride=2, pad_lo=1, act='relu', rar=True,
         res='bf16'),
    case(C, 'conv BN128 s2 t1x8x16 e0', F=2, H=32, W=32, Cin=64, N=128, stride=2, pad_lo=1, act='relu', rar=True,
         res='bf16', out='f32'),
    case(C, 'conv BN64 s1 t2x8x8 e0', F=3, H=8, W=8, Cin=64, N=64, act='relu', rar=True, res='bf16', out='f32'),
    case(C, 'halo3 BN64 e0 r1', F=2, H=16, W=16, Cin=64, N=64, act='relu', rar=True, res='bf16', ooff=1, opad=8),
    # ---------------- stride-2 3x3 at 64 x 192 (output 32 x 96: 64-column tiles, ragged), pad_lo 0 and 1; 1x1 s2
    *[case(C, 'conv BN%d s2 t1x2x64 e1' % (64 if n == 64 else 128), F=2, H=64, W=192, Cin=64, N=n, stride=2, pad_lo=p,
           act=a) for (n, p, a) in [(64, 0, 'none'), (64, 1, 'silu'), (128, 0, 'none'), (128, 1, 'relu')]],
    case(C, 'conv BN128 s2 t1x8x16 e1', F=2, H=32, W=32, Cin=64, N=128, stride=2, pad_lo=0, gn=True),
    case(C, 'conv BN128 s2 t2x8x8 e1', F=3, H=16, W=16, Cin=64, N=128, ksize=1, stride=2, pad_lo=0),
    case(C, 'conv BN128 s2 t4x4x8 e1', F=3, H=8, W=16, Cin=64, N=128, ksize=1, stride=2, pad_lo=0, out='f32'),
    # stride 2 on an input channel slice: NaN in [Cin, ldx)
    case(C, 'conv BN64 s2 t1x8x16 e1', F=2, H=32, W=32, Cin=64, N=64, stride=2, pad_lo=0, xpad=64),
    case(C, 'conv BN128 s2 t1x8x16 e1', F=2, H=32, W=32, Cin=128, N=128, stride=2, pad_lo=1, xpad=64, res='bf16'),
    case(C, 'conv BN128 s2 t2x8x8 e1', F=3, H=16, W=16, Cin=64, N=128, ksize=1, stride=2, pad_lo=0, xpad=64),
    # ---------------- multi-frame tiles (tn > 1), F % tn != 0: residual (TMA and direct), NCHW output
    case(C, 'conv BN128 s1 t2x8x8 e1', F=3, H=8, W=8, Cin=64, N=128, res='bf16', act='gelu'),
    case(C, 'conv BN128 s1 t2x8x8 e0', F=3, H=8, W=8, Cin=64, N=128, res='bf16', out='f32'),
    case(C, 'conv BN128 s1 t2x8x8 e0', F=3, H=8, W=8, Cin=64, N=128, res='f32', ooff=1, opad=8),
    case(C, 'conv BN64 s1 t8x4x4 e0', F=3, H=4, W=4, Cin=64, N=64, res='bf16', out='f32', act='silu'),
    case(C, 'conv BN128 s1 t8x4x4 e1', F=5, H=4, W=4, Cin=256, N=256, res='f32', out='f32'),
    case(C, 'conv BN64 s1 t2x8x8 e0', F=3, H=8, W=8, Cin=64, N=3, out='nchw'),
    case(C, 'conv BN128 s1 t2x8x8 e0', F=3, H=8, W=8, Cin=64, N=128, out='nchw', act='lrelu'),
    case(C, 'halo3 BN64 e0 r1', F=2, H=16, W=16, Cin=64, N=3, out='nchw'),
    # ---------------- channel tails and slices on stride-1 convs
    case(C, 'conv BN128 s1 t1x8x16 e1', F=2, H=8, W=16, Cin=96, N=96, xpad=8, res='bf16', rpad=32),
    case(C, 'halo3 BN64 e1 r0', F=2, H=16, W=16, Cin=160, N=64, xpad=32, res='bf16'),
    case(C, 'conv BN128 s1 t1x16x8 e1', F=2, H=16, W=8, Cin=64, N=256, ksize=1, pad_lo=0, res='bf16', opad=64),
    # ---------------- out aliasing the residual (bf16): halo and non-halo
    case(C, 'halo3 BN64 e1 r1', F=2, H=16, W=16, Cin=64, N=64, res='bf16', alias=True),
    case(C, 'conv BN128 s1 t1x4x32 e1', F=2, H=32, W=32, Cin=64, N=256, res='bf16', alias=True, act='silu'),
    # ---------------- the fixed cases: bf16 output offset by one element (ldo % 8 == 0), bias offset by one float
    case(C, 'conv BN128 s1 t1x4x32 e0', F=2, H=32, W=32, Cin=64, N=256, ooff=1, opad=8, act='gelu'),
    case(C, 'halo3 BN64 e0 r1', F=2, H=16, W=16, Cin=64, N=64, ooff=1, opad=8),
    case(C, 'halo3 BN128 e0 r0', F=2, H=16, W=16, Cin=64, N=128, ooff=1, opad=16, res='bf16'),
    case(C, 'conv BN128 s1 t1x4x32 e1', F=2, H=32, W=32, Cin=64, N=256, boff=1, act='relu'),
    case(C, 'halo3 BN128 e1 r0', F=2, H=16, W=16, Cin=64, N=128, boff=1),
    case(C, 'conv BN128 s1 t1x4x32 e1', F=2, H=32, W=32, Cin=64, N=256, boff=1, sft=0.7, res='bf16'),
    # ---------------- 256-wide conv tiles, sized to fill every SM
    case(C, 'conv BN256 s1 t1x4x32 e1', wide=True, H=32, W=32, Cin=64, N=256, act='gelu', res='bf16'),
    case(C, 'conv BN256 s1 t1x4x32 e0', wide=True, H=32, W=32, Cin=64, N=256, res='bf16', out='f32', boff=1),
    # ---------------- upsample-folded conv (four phase launches)
    case(U, 'halo3 BN64 e1 r1', F=2, H=16, W=16, Cin=64, N=64, act='silu'),
    case(U, 'halo3 BN128 e1 r0', F=2, H=16, W=8, Cin=128, N=128, boff=1),
    case(U, 'conv BN128 s1 t2x8x8 e1', F=3, H=8, W=8, Cin=64, N=256, out='f32'),
    # ---------------- RGB stem, bias offset by one float
    case(R, 'rgb_conv 3x3/1 N64', F=2, H=16, W=16, N=64, ksize=3, stride=1, pad_lo=1, boff=1, act='relu', opad=8),
    case(R, 'rgb_conv 7x7/2 N64', F=2, H=32, W=32, N=64, ksize=7, stride=2, pad_lo=3, boff=1),
    case(R, 'rgb_conv 3x3/1 N128', F=2, H=16, W=16, N=128, ksize=3, stride=1, pad_lo=1, boff=1, act='relu'),
    case(R, 'rgb_conv 3x3/1 N64', F=2, H=16, W=16, N=64, ksize=3, stride=1, pad_lo=1),
]

# (launch pattern, feature) pairs the case matrix must keep covering (features() names the features of a case)
REQUIRED = [
    (r'conv BN128 s1 \S+ e1', 'sft256'), (r'conv BN128 s1 \S+ e1', 'sft256+gn'),
    (r'conv BN128 s1 \S+ e1', 'sft512'), (r'conv BN128 s1 \S+ e1', 'sft512+gn'),
    (r'conv BN128 s1 \S+ e1', 'sft+ragged'), (r'conv BN64 s1 t[2-9]x', 'sft+ftail'),
    (r' e0', 'sft+f32'), (r' e0', 'sft+aoff'),
    *[(k, 'act:' + a) for k in ('linear ', 'conv ', 'halo3 ') for a in ACT_CODE],
    (r'linear BN(64|128) e1', 'act:sigmoid+fewrows'),
    (r'linear ', 'res:bf16>f32'), (r'linear ', 'res:f32>bf16'), (r'conv ', 'res:bf16>f32'), (r'conv ', 'res:f32>bf16'),
    (r'conv BN\d+ s2 ', 'rar'), (r' e0', 'rar'),
    (r'conv BN\d+ s2 t1x2x64 ', 'pad0+ragged'), (r'conv BN\d+ s2 t1x2x64 ', 'pad1+ragged'), (r'conv BN\d+ s2 ', 'k1'),
    (r'conv BN\d+ s2 ', 'xslice'),
    (r'conv BN\d+ s1 t[2-9]x\S+ e1', 'ftail+res'), (r'conv BN\d+ s1 t[2-9]x\S+ e0', 'ftail+res'),
    (r'conv BN\d+ s1 t[2-9]x', 'nchw'),
    *[(r'linear ', 'M%d' % m) for m in (1, 127, 129)], *[(r'linear ', 'N%d' % n) for n in (3, 40, 200)],
    (r'linear ', 'ktail'), (r'linear BN256 ', 'ntail'),
    (r'halo3 ', 'alias:bf16'), (r'conv ', 'alias:bf16'),
    (r'conv BN\d+ \S+ \S+ e0', 'ooff1'), (r'linear BN\d+ e0', 'ooff1'), (r'halo3 BN\d+ e0', 'ooff1'),
    (r'linear ', 'boff1'), (r'conv ', 'boff1'), (r'halo3 ', 'boff1'), (r'rgb_conv ', 'boff1'),
    (r'conv BN256 ', ''), (r'halo3 BN64 e1 r1', ''), (r'halo3 BN128 e1 r0', ''), (r'conv BN64 ', ''),
]


def features(c):
    """The properties of a case that REQUIRED names."""
    f = {''}
    if c['sft'] is not None:
        f.add('sft%d' % c['N'] + ('+gn' if c['gn'] else ''))
        if c['entry'] == 'conv' and (c['W'] // c['stride']) % 32:
            f.add('sft+ragged')
        if c['F'] % 2:
            f.add('sft+ftail')
        if c['out'] == 'f32':
            f.add('sft+f32')
        if c['aoff']:
            f.add('sft+aoff')
    f.add('act:' + c['act'])
    if c['act'] == 'sigmoid' and c['entry'] == 'linear' and c['M'] <= 8 and c['N'] in (128, 256):
        f.add('act:sigmoid+fewrows')
    if c['res'] is not None and c['res'] != c['out']:
        f.add('res:%s>%s' % (c['res'], c['out']))
    if c['rar']:
        f.add('rar')
    if c['stride'] == 2 and c['entry'] == 'conv':
        f.add('pad%d+ragged' % c['pad_lo'])
        if c['ksize'] == 1:
            f.add('k1')
        if c['xpad']:
            f.add('xslice')
    if c['entry'] == 'conv' and c['F'] % 2 and c['res'] is not None:
        f.add('ftail+res')
    if c['out'] == 'nchw':
        f.add('nchw')
    if c['entry'] == 'linear':
        f.add('M%d' % c['M'])
        f.add('N%d' % c['N'])
        if c['K'] % 64 and c['kpad']:
            f.add('ktail')
        if c['N'] % 256:
            f.add('ntail')
    if c['alias']:
        f.add('alias:' + c['out'])
    if c['ooff'] == 1 and c['out'] == 'bf16' and (c['N'] + c['opad']) % 8 == 0:
        f.add('ooff1')
    if c['boff'] == 1 and c['N'] % 32 == 0:
        f.add('boff1')
    return f


def test_cases_cover_the_required_paths():
    """Every (launch, feature) pair of REQUIRED is the pinned launch and a feature of some case."""
    missing = [(pat, feat) for pat, feat in REQUIRED
               if not any(re.search(pat, c['launch']) and feat in features(c) for c in CASES)]
    assert not missing, missing
    ids = [case_id(c) for c in CASES]
    assert len(set(ids)) == len(ids), [i for i in ids if ids.count(i) > 1]


# ------------------------------------------------------------------------------------------------ machinery
def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _uniform(shape, g, lo, hi):
    return torch.rand(shape, generator=g, device=DEV, dtype=torch.float64) * (hi - lo) + lo


def _nan(n, dtype):
    return torch.full((n,), float('nan'), dtype=dtype, device=DEV)


def _strides(shape, ld):
    st, s = [1], ld
    for d in reversed(shape[:-1]):
        st.insert(0, s)
        s *= d
    return st


class Buf:
    """A NaN-poisoned flat buffer holding one channels-last view [..., C] with row pitch ld at element offset off,
    followed by one more row of poison."""

    def __init__(self, shape, dtype, ld, off, data=None, contiguous_view=False):
        rows = math.prod(shape[:-1])
        self.buf = _nan(off + (rows + 1) * ld, dtype)
        if contiguous_view:
            self.view = self.buf[off:off + math.prod(shape)].view(*shape)
        else:
            self.view = self.buf.as_strided(shape, _strides(shape, ld), off)
        if data is not None:
            self.view.copy_(data)
        self.mask = torch.zeros(self.buf.numel(), dtype=torch.bool, device=DEV)
        self.mask.as_strided(self.view.shape, self.view.stride(), self.view.storage_offset()).fill_(True)
        self.before = self.buf.clone()

    def bits(self, t):
        return t.view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)

    def untouched(self):
        """Elements outside the view are bit-identical to what they were before the call."""
        return torch.equal(self.bits(self.buf)[~self.mask], self.bits(self.before)[~self.mask])


def launch_key(desc):
    t = desc.split()
    if t[0] == 'rgb_conv':
        return desc.strip()
    kind = 'conv' if re.match(r'conv\d$', t[0]) else t[0]
    order = ('BN', 's', 't', 'e', 'r')                  # kernel, BN, mode, tile, epilogue path, resident weights
    keep = [x for x in t[1:] if re.match(r'(BN\d+|s\d|t\d+x\d+x\d+|e\d|r\d)$', x)]
    keep.sort(key=lambda x: order.index('BN' if x.startswith('BN') else x[0]))
    return ' '.join([kind] + keep)


def launches(fn, tmp_path):
    """Runs fn under the library's launch profiler -> the GEMM-class launch descriptions."""
    from pgtformer_b200 import ops
    path = os.path.join(str(tmp_path), 'launches.csv')
    ops.profile_begin()
    fn()
    ops.profile_end(path)
    with open(path) as fh:
        return [r['desc'] for r in csv.DictReader(fh) if r['class'] == '0']


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def resolve(c):
    """Sizes of the 256-wide cases from the SM count: enough 128 x 256 tiles to occupy every SM."""
    c = dict(c)
    if c['wide'] and c['entry'] == 'linear':
        c['M'] = 128 * -(-_sms() // 2) - 5              # ragged last row tile, two n-tiles per row tile
    elif c['wide']:
        c['F'] = -(-_sms() * 128 // (c['H'] * c['W']))
    return c


def _pad_conv(c):
    k, s, p = c['ksize'], c['stride'], c['pad_lo']
    if s == 1:
        return (1, 1, 1, 1) if k == 3 else (0, 0, 0, 0)
    if k == 1:
        return (0, 0, 0, 0)
    return (0, 1, 0, 1) if p == 0 else (1, 1, 1, 1)


def run_case(c, tmp_path, seed=0):
    """Builds the poisoned operands of case c, runs it under the profiler -> (output Buf, got [..., N] in NHWC order,
    fp64 reference, fp64 S, launch keys, gn statistics Buf or None, tile (th, tw) of the launch)."""
    from pgtformer_b200 import ops
    from pgtformer_b200.engine import _pack_conv, _pack_rgb, _pack_up2x
    g = _gen(1000 + seed)
    N = c['N']
    chs = torch.exp2(_uniform((N,), g, -6, 6))                          # per-output-channel scale
    entry = c['entry']
    bf16 = torch.bfloat16
    # ---- operands, reference accumulation z and its magnitude sum Sa (both without bias)
    if entry == 'linear':
        M, K = c['M'], c['K']
        a = (torch.randn(M, K, generator=g, device=DEV, dtype=torch.float64) *
             torch.exp2(_uniform((M, 1), g, -2, 2))).to(bf16)
        w = (torch.randn(N, K, generator=g, device=DEV, dtype=torch.float64) * chs[:, None] * K ** -0.5).to(bf16)
        lda = ldw = K + c['kpad'] if c['kpad'] else (K + 7) // 8 * 8
        A = Buf((M, K), bf16, lda, 0, a)
        Wb = Buf((N + 1, K), bf16, ldw, 0)
        Wb.view[:N].copy_(w)
        Wb.before = Wb.buf.clone()
        wview = Wb.view[:N]
        z = a.double() @ w.double().t()
        Sa = a.double().abs() @ w.double().abs().t()
        oshape = (M, N)
        keep = [A, Wb]
    elif entry == 'rgb':
        Fr, H, W, k = c['F'], c['H'], c['W'], c['ksize']
        x = torch.rand(Fr, 3, H, W, generator=g, device=DEV, dtype=torch.float64).float()
        w = (torch.randn(N, 3, k, k, generator=g, device=DEV, dtype=torch.float64) * chs[:, None, None, None] *
             (3 * k * k) ** -0.5).to(bf16).float()
        wp = _pack_rgb(w)
        wview = wp
        xr = x.to(bf16).double()
        pd = c['pad_lo']
        z = F.conv2d(xr, w.double(), stride=c['stride'], padding=pd).permute(0, 2, 3, 1)
        Sa = F.conv2d(xr.abs(), w.double().abs(), stride=c['stride'], padding=pd).permute(0, 2, 3, 1)
        oshape = tuple(z.shape)
        keep = []
    else:
        Fr, H, W, Cin, k = c['F'], c['H'], c['W'], c['Cin'], c['ksize']
        x = (torch.randn(Fr, H, W, Cin, generator=g, device=DEV, dtype=torch.float64) *
             torch.exp2(_uniform((Fr, H, W, 1), g, -2, 2))).to(bf16)
        X = Buf((Fr, H, W, Cin), bf16, Cin + c['xpad'], 0, x)
        x64 = x.double().permute(0, 3, 1, 2)
        w = (torch.randn(N, Cin, 3, 3, generator=g, device=DEV, dtype=torch.float64)[:, :, :k, :k] *
             chs[:, None, None, None] * (k * k * Cin) ** -0.5).to(bf16).float()
        if entry == 'up2x':
            wp = _pack_up2x(w)                                           # [4, N, 4 * CinPad], rounded once more
            cp = wp.shape[2] // 4
            wview = wp
            z = torch.empty(Fr, N, 2 * H, 2 * W, dtype=torch.float64, device=DEV)
            Sa = torch.empty_like(z)
            for ph in range(4):
                py, px = ph >> 1, ph & 1
                wph = wp[ph].double().view(N, 2, 2, cp)[..., :Cin].permute(0, 3, 1, 2)
                xp = F.pad(x64, (1 - px, px, 1 - py, py))
                z[:, :, py::2, px::2] = F.conv2d(xp, wph)
                Sa[:, :, py::2, px::2] = F.conv2d(xp.abs(), wph.abs())
            oshape = (Fr, 2 * H, 2 * W, N)
        else:
            wp = _pack_conv(w)
            Wb = Buf((N + 1, wp.shape[1]), bf16, wp.shape[1] + 8, 0)
            Wb.view[:N].copy_(wp)
            Wb.before = Wb.buf.clone()
            wview = Wb.view[:N]
            keep_w = [Wb]
            xp = F.pad(x64, _pad_conv(c))
            z = F.conv2d(xp, w.double(), stride=c['stride'])
            Sa = F.conv2d(xp.abs(), w.double().abs(), stride=c['stride'])
            oshape = (Fr, H // c['stride'], W // c['stride'], N)
        z = z.permute(0, 2, 3, 1)
        Sa = Sa.permute(0, 2, 3, 1)
        keep = [X] + (keep_w if entry == 'conv' else [])
    # ---- bias, residual, scale
    b = bv = None
    if c['bias']:
        b = (torch.randn(N, generator=g, device=DEV, dtype=torch.float64) * chs * 0.5).float()
        Bb = Buf((N,), torch.float32, N, c['boff'], b)
        bv = Bb.view
        keep.append(Bb)
        z = z + b.double()
        Sa = Sa + b.double().abs()
    rows_scale = torch.exp2(_uniform(oshape[:-1] + (1,), g, -1, 1))
    res = rv = None
    if c['res'] is not None:
        rdt = bf16 if c['res'] == 'bf16' else torch.float32
        res = (torch.randn(oshape, generator=g, device=DEV, dtype=torch.float64) * chs * rows_scale).to(rdt)
        Rb = Buf(oshape, rdt, N + c['rpad'], c['roff'], res)
        rv = Rb.view
        keep.append(Rb)
    sv = None
    if c['sft'] is not None:
        s = torch.randn(oshape, generator=g, device=DEV, dtype=torch.float64).to(bf16)
        Sb = Buf(oshape, bf16, N + c['apad'], c['aoff'], s)
        sv = Sb.view
        keep.append(Sb)
    # ---- output
    odt = bf16 if c['out'] == 'bf16' else torch.float32
    if c['alias']:
        Ob = Rb
        assert Ob.view.dtype == odt
    elif c['out'] == 'nchw':
        Ob = Buf((oshape[0], N, oshape[1], oshape[2]), odt, oshape[2], c['ooff'], contiguous_view=True)
    else:
        Ob = Buf(oshape, odt, N + c['opad'], c['ooff'])
    Gb = None
    if c['gn']:
        Gb = Buf((math.prod(oshape[:-1]) // 32, 32, 2), torch.float32, 2, 0, contiguous_view=True)
    act = ACT_CODE[c['act']]

    def call():
        if entry == 'linear':
            ops.linear(A.view, wview, Ob.view, bias=bv, act=act, residual=rv, relu_after_res=c['rar'],
                       gn_stats=Gb.view if Gb else None)
        elif entry == 'conv':
            ops.conv(X.view, wview, N, Ob.view, ksize=c['ksize'], stride=c['stride'], pad_lo=c['pad_lo'], bias=bv,
                     act=act, residual=rv, sft_scale=sv, sft_w=c['sft'] or 0.0, nchw=c['out'] == 'nchw',
                     relu_after_res=c['rar'], gn_stats=Gb.view if Gb else None)
        elif entry == 'up2x':
            ops.conv_up2x(X.view, wview, N, Ob.view, bias=bv, act=act)
        else:
            ops.conv_rgb(x, wview, bv, Ob.view, c['ksize'], c['stride'], c['pad_lo'], act=act)

    keys = [launch_key(d) for d in launches(call, tmp_path)]
    torch.cuda.synchronize()
    # ---- fp64 epilogue and magnitude sums
    if c['sft'] is not None:
        r, sw = res.double(), float(c['sft'])
        s64 = s.double()
        ref = r + sw * (r * s64 + z)
        S = abs(sw) * Sa + r.abs() + abs(sw) * (r * s64).abs()
    elif c['rar']:
        ref = F.relu(z + res.double())
        S = Sa + res.double().abs()
    else:
        ref = _act(z, c['act'])
        S = Sa * (1.2 if c['act'] in SMOOTH else 1.0) + (ref.abs() if c['act'] in SMOOTH else 0)
        if res is not None:
            ref = ref + res.double()
            S = S + res.double().abs()
    got = Ob.view.permute(0, 2, 3, 1) if c['out'] == 'nchw' else Ob.view
    return dict(out=Ob, got=got, ref=ref, S=S, keys=keys, gn=Gb, keep=keep)


def family(keys):
    return keys[0].split()[0]


def check_bound(got, ref, S, bf16_out, fam, what):
    got = got.double()
    assert torch.isfinite(got).all(), '%s: %d non-finite outputs' % (what, int((~torch.isfinite(got)).sum()))
    excess = (got - ref).abs() - (U_BF16 * ref.abs() if bf16_out else 0)
    ratio = excess / S.clamp_min(1e-300)
    worst = ratio.max().item()
    WORST[fam] = max(WORST.get(fam, 0.0), worst)
    bad = ratio > EPS[fam]
    if bad.any():
        i = tuple(int(v) for v in (ratio == ratio.max()).nonzero()[0])
        raise AssertionError('%s: %d of %d elements beyond the bound; worst err / S = 2^%.1f (eps 2^%.0f) at %s: '
                             'got %r ref %r S %r' % (what, int(bad.sum()), bad.numel(), math.log2(worst), math.log2(EPS[fam]),
                                              i, got[i].item(), ref[i].item(), S[i].item()))


def check_gn(r, c, th, tw, what):
    """Fused statistics of every (tile, quadrant, group) against fp64 sums of the stored bf16 output (the bound of
    test_gn_stats_gpu.py: the epilogue sums the fp32 values before their bf16 rounding, in fp32 over <= 1024 terms)."""
    Gb = r['gn']
    assert Gb.untouched()
    st = Gb.view.double()
    assert torch.isfinite(st).all(), what + ': non-finite statistics'
    x = r['got'].double()
    N = x.shape[-1]
    if c['entry'] == 'linear':
        v = x.reshape(-1, 4, 32, 32, N // 32)                            # [tile][quadrant][row][group][channel]
    else:
        Fr, H, W, _ = x.shape
        v = x.reshape(Fr, H // th, th, W // tw, tw, N).permute(0, 1, 3, 2, 4, 5).reshape(-1, 4, 32, 32, N // 32)
    got = st.view(-1, 4, 32, 2)
    for k, (ref, allowed) in enumerate(((v.sum((2, 4)), (2.0 ** -8 + 2.0 ** -13) * v.abs().sum((2, 4))),
                                        (v.pow(2).sum((2, 4)), (2.0 ** -7 + 2.0 ** -13) * v.pow(2).sum((2, 4))))):
        bad = (got[..., k] - ref).abs() > allowed
        assert not bad.any(), '%s: %d %s statistics beyond the bound' % (what, int(bad.sum()), ('sum', 'sumsq')[k])


@gpu
@pytest.mark.parametrize('c', CASES, ids=case_id)
def test_epilogue(c, tmp_path):
    c = resolve(c)
    what = case_id(c)
    r = run_case(c, tmp_path)
    nlaunch = 4 if c['entry'] == 'up2x' else 1
    assert r['keys'] == [c['launch']] * nlaunch, (what, r['keys'])
    assert r['out'].untouched(), what + ': elements outside the output view were written'
    for b in r['keep']:
        assert b.untouched(), what + ': an input buffer was written'
    check_bound(r['got'], r['ref'], r['S'], c['out'] == 'bf16', family(r['keys']), what)
    if c['gn']:
        m = re.search(r' t1x(\d+)x(\d+) ', r['keys'][0] + ' ')
        th, tw = (int(m.group(1)), int(m.group(2))) if m else (16, 8)
        check_gn(r, c, th, tw, what)


# ------------------------------------------------------------------------------------------------ identities
IDENTITY = [
    dict(entry=L, M=300, N=256, K=192, fast='linear BN128 e1', direct='linear BN128 e0'),
    dict(entry=L, M=129, N=64, K=200, fast='linear BN64 e1', direct='linear BN64 e0'),
    dict(entry=C, F=2, H=8, W=16, Cin=64, N=96, fast='conv BN128 s1 t1x8x16 e1', direct='conv BN128 s1 t1x8x16 e0'),
    dict(entry=C, F=3, H=8, W=8, Cin=64, N=64, fast='conv BN64 s1 t2x8x8 e1', direct='conv BN64 s1 t2x8x8 e0'),
    dict(entry=C, F=2, H=16, W=16, Cin=64, N=64, fast='halo3 BN64 e1 r1', direct='halo3 BN64 e0 r1'),
    dict(entry=C, F=2, H=24, W=40, Cin=64, N=128, fast='halo3 BN128 e1 r0', direct='halo3 BN128 e0 r0'),
]


@gpu
@pytest.mark.parametrize('act', ['none', 'relu', 'lrelu'])
@pytest.mark.parametrize('out,res', [('bf16', None), ('bf16', 'bf16'), ('f32', 'f32')])
@pytest.mark.parametrize('shape', IDENTITY, ids=lambda s: '%s-N%d-%s' % (s['entry'], s['N'], s['fast'].split()[0]))
def test_tma_store_path_equals_direct_path(shape, out, res, act, tmp_path):
    """The same plain epilogue through the TMA-store path (ldo = N) and the direct path (a row pitch that is not a
    multiple of 16 bytes, and a view offset by one element): identical bits."""
    base = {k: v for k, v in shape.items() if k not in ('fast', 'direct', 'entry')}
    pad = 4 if out == 'bf16' else 2
    got = []
    for opad, ooff, want in ((0, 0, shape['fast']), (pad, 0, shape['direct']), (pad * 2, 1, shape['direct'])):
        c = case(shape['entry'], want, act=act, out=out, res=res, opad=opad, ooff=ooff, **base)
        r = run_case(c, tmp_path, seed=7)
        assert r['keys'] == [want], r['keys']
        assert r['out'].untouched()
        check_bound(r['got'], r['ref'], r['S'], out == 'bf16', family(r['keys']), case_id(c))
        got.append(r['got'].clone())
    assert torch.equal(got[0], got[1]) and torch.equal(got[0], got[2])


@gpu
@pytest.mark.parametrize('out,res', [('bf16', 'bf16'), ('f32', None)])
def test_linear_64_column_slices_equal_one_launch(out, res, tmp_path):
    """A linear launched as 64-column slices (gemm_tc_kernel<64>) and as one BN = 128 launch: identical bits, since both
    accumulate every output element's k-blocks in the same order."""
    from pgtformer_b200 import ops
    g = _gen(5)
    M, N, K = 1000, 256, 520
    a = torch.randn(M, K, generator=g, device=DEV).to(torch.bfloat16)
    w = (torch.randn(N, K, generator=g, device=DEV) * torch.exp2(torch.rand(N, 1, generator=g, device=DEV) * 12 - 6) *
         K ** -0.5).to(torch.bfloat16)
    b = torch.randn(N, generator=g, device=DEV)
    odt = torch.bfloat16 if out == 'bf16' else torch.float32
    r = torch.randn(M, N, generator=g, device=DEV).to(odt) if res else None
    one = torch.full((M, N), float('nan'), dtype=odt, device=DEV)
    sl = torch.full((M, N), float('nan'), dtype=odt, device=DEV)
    keys = [launch_key(d) for d in launches(
        lambda: ops.linear(a, w, one, bias=b, act=ops.ACT_GELU, residual=r), tmp_path)]
    assert keys == ['linear BN128 e1'], keys

    def slices():
        for n0 in range(0, N, 64):
            ops.linear(a, w[n0:n0 + 64], sl[:, n0:n0 + 64], bias=b[n0:n0 + 64], act=ops.ACT_GELU,
                       residual=r[:, n0:n0 + 64] if r is not None else None)
    keys = [launch_key(d) for d in launches(slices, tmp_path)]
    assert keys == ['linear BN64 e1'] * (N // 64), keys
    assert torch.isfinite(one).all() and torch.equal(one, sl)


@pytest.fixture(scope='module', autouse=True)
def _report_worst():
    yield
    if WORST:
        print('\nworst err / S per kernel family: ' + ', '.join(
            '%s %s (eps 2^%.0f)' % (k, '2^%.1f' % math.log2(v) if v > 0 else 'within the bf16 rounding',
                                    math.log2(EPS[k]))
            for k, v in sorted(WORST.items())))
