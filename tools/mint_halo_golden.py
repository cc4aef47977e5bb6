"""Records outputs and fused GroupNorm statistics of the Cout <= 128 halo convs (`conv_halo_kernel<BN, false>`) on
seeded inputs, for tests/test_halo_pingpong_gpu.py: run with the library as it was before the ping-pong schedule, so
the test shows the new schedule computes the same bits.

tests/golden/halo_pingpong_outputs.pt was recorded on an H100 with the library built at commit
f8b20dc3b74f0aea776a94afd2561131ccf08fdd (the commit before the ping-pong schedule); the file stores that id as
`library_commit`.  To reproduce it, check out that commit, build it, and run this script from the newer tree with the
old package first on the path:

    PYTHONPATH=<old checkout> python tools/mint_halo_golden.py OUT.pt --commit <id of the old checkout>

Each case keeps a strided sample of every tensor (the `conftest.golden_sample` format: `<key>`, `<key>_shape`,
`<key>_stride`) so the file stays small.
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.append(ROOT)

# kind, F, H, W, Cin, Cout, and the epilogue.  res / out: dtype of the residual / output ('nchw': fp32 NCHW); sft: the
# residual is modulated by a bf16 scale; slice: output into channels [32, 32 + Cout) of a wider buffer.  16 x 8-pixel
# tiles: 37 x 29 -> 3 x 4 per frame; 112 x 152 -> 133 (one more than the H100's 132 SMs);
# 5 x 16 x 424 -> 265 (CTA 0 takes three tiles, the others two).
CASES = (
    dict(name='c32_ragged', kind='conv', F=1, H=37, W=29, Cin=64, Cout=32, act='silu'),
    dict(name='c48_cin8_133tiles', kind='conv', F=1, H=112, W=152, Cin=8, Cout=48, act='lrelu', res='bf16'),
    dict(name='c64_265tiles_gn', kind='conv', F=5, H=16, W=424, Cin=64, Cout=64, res='bf16', gn=True),
    dict(name='c64_cin128_f32res_f32out', kind='conv', F=2, H=40, W=44, Cin=128, Cout=64, act='gelu', res='f32', out='f32'),
    dict(name='c64_f32res_bf16out_relu_after', kind='conv', F=2, H=37, W=29, Cin=64, Cout=64, act='relu', res='f32',
         relu_after_res=True),
    dict(name='c64_sft', kind='conv', F=2, H=37, W=29, Cin=64, Cout=64, res='bf16', sft=True),
    dict(name='c96_nchw', kind='conv', F=2, H=37, W=45, Cin=128, Cout=96, act='silu', out='nchw'),
    dict(name='c128_sft', kind='conv', F=3, H=48, W=40, Cin=128, Cout=128, res='bf16', sft=True),
    dict(name='c128_cin288_gn', kind='conv', F=3, H=64, W=64, Cin=288, Cout=128, gn=True),
    dict(name='c128_slice_133tiles', kind='conv', F=1, H=112, W=152, Cin=64, Cout=128, act='silu', slice=True),
    dict(name='c128_res_265tiles', kind='conv', F=5, H=16, W=424, Cin=128, Cout=128, res='bf16', gn=True),
    dict(name='up2x_c64_gn', kind='up2x', F=3, H=32, W=24, Cin=64, Cout=64, gn=True),
    dict(name='up2x_c128_resident_gn', kind='up2x', F=2, H=40, W=40, Cin=64, Cout=128, gn=True),
    dict(name='up2x_c128_streamed_gn', kind='up2x', F=2, H=20, W=36, Cin=128, Cout=128, gn=True),
)
SAMPLES = 4096          # about this many elements kept per tensor


def rnd(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to('cuda')


def run_case(c, seed=1000):
    """Runs case c through the ctypes binding -> {key: full result tensor}."""
    from pgtformer_b200 import ops
    from pgtformer_b200.engine import _pack_conv, _pack_up2x
    acts = {'silu': ops.ACT_SILU, 'lrelu': ops.ACT_LRELU02, 'gelu': ops.ACT_GELU, 'relu': ops.ACT_RELU}
    act = acts[c['act']] if 'act' in c else ops.ACT_NONE
    F, H, W, Cin, N = c['F'], c['H'], c['W'], c['Cin'], c['Cout']
    x = rnd((F, H, W, Cin), seed).to(torch.bfloat16)
    w = rnd((N, Cin, 3, 3), seed + 1, (9 * Cin) ** -0.5)
    b = rnd((N,), seed + 2, 0.1)
    up = c['kind'] == 'up2x'
    Ho, Wo = (2 * H, 2 * W) if up else (H, W)
    odt = torch.float32 if c.get('out') in ('f32', 'nchw') else torch.bfloat16
    res = {'bf16': torch.bfloat16, 'f32': torch.float32}.get(c.get('res'))
    res = rnd((F, Ho, Wo, N), seed + 3).to(res) if res is not None else None
    stats = None
    if c.get('gn'):
        tpf = ops.conv_tiles_per_frame(H, W, N, 2, 1, 1) if up else ops.conv_tiles_per_frame(H, W, N)
        assert tpf > 0
        stats = torch.zeros((16 if up else 4) * F * tpf * 64, device='cuda')
    if up:
        out = torch.empty(F, Ho, Wo, N, dtype=odt, device='cuda')
        ops.conv_up2x(x, _pack_up2x(w), N, out, bias=b, act=act, gn_stats=stats)
        full = out
    elif c.get('out') == 'nchw':
        out = full = torch.empty(F, N, H, W, dtype=odt, device='cuda')
        ops.conv(x, _pack_conv(w), N, out, bias=b, act=act, residual=res, nchw=True)
    else:
        full = torch.zeros(F, H, W, N + 96, dtype=odt, device='cuda') if c.get('slice') else None
        out = full[..., 32:32 + N] if full is not None else torch.empty(F, H, W, N, dtype=odt, device='cuda')
        full = full if full is not None else out
        sft = rnd((F, H, W, N), seed + 4).to(torch.bfloat16) if c.get('sft') else None
        ops.conv(x, _pack_conv(w), N, out, bias=b, act=act, residual=res, sft_scale=sft, sft_w=0.7 if sft is not None else 0.0,
                 relu_after_res=c.get('relu_after_res', False), gn_stats=stats)
    torch.cuda.synchronize()
    r = {'out': full}
    if stats is not None:
        r['stats'] = stats
    return r


def sample(t):
    """-> (flat strided sample as fp32 on the CPU, stride): odd strides reach every channel."""
    n = t.numel()
    s = max(1, n // SAMPLES) | 1
    return t.float().cpu().reshape(-1)[::s].clone(), s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('out')
    ap.add_argument('--commit', required=True, help='commit the loaded library was built from')
    args = ap.parse_args()
    cases = []
    for c in CASES:
        rec = {'case': dict(c)}
        for k, t in run_case(c).items():
            rec[k], rec[k + '_stride'] = sample(t)
            rec[k + '_shape'] = tuple(t.shape)
        cases.append(rec)
    torch.save({'cases': cases, 'library_commit': args.commit}, args.out)


if __name__ == '__main__':
    main()
