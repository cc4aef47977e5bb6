"""Micro-benchmark of single conv shapes (CUDA events, 20 reps).  The wide cases (Cout > 128, the flagship workload's
own shapes at 16 clips = 48 frames) time the launch dispatch_gemm picks against the same conv launched as 128-channel
slices, which take the library's Cout <= 128 path (the halo kernel for stride-1 3x3 and upsample-phase convs,
gemm_tc_kernel<128> otherwise): both in one process, with no switch in the library.  `python tools/micro_conv.py wide`.
`python tools/micro_conv.py halo` times each Cout <= 128 halo-kernel shape of the flagship workload alone."""
import os
import sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pgtformer_b200 import ops  # noqa: E402
from pgtformer_b200.engine import _pack_conv, _pack_up2x  # noqa: E402

dev = 'cuda'


def timeit(fn, reps=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def conv_case(F, H, C, N, residual, out_dtype=torch.bfloat16, act=0):
    x = torch.randn(F, H, H, C, device=dev).bfloat16()
    w = _pack_conv(torch.randn(N, C, 3, 3, device=dev) * 0.05)
    b = torch.zeros(N, device=dev)
    res = torch.randn(F, H, H, N, device=dev).to(out_dtype) if residual else None
    out = torch.empty(F, H, H, N, device=dev, dtype=out_dtype)
    ms = timeit(lambda: ops.conv(x, w, N, out, bias=b, residual=res, act=act))
    fl = 2.0 * F * H * H * N * 9 * C
    print('conv F%d H%d C%d N%d res=%d %s act=%d: %.3f ms  %.0f TF/s' % (F, H, C, N, residual, str(out_dtype)[6:], act, ms, fl / ms / 1e9))


def wide_case(name, flops, run, N):
    """run(n0, n1) launches output channels [n0, n1)."""
    def sliced():
        for n0 in range(0, N, 128):
            run(n0, min(N, n0 + 128))
    ms_d, ms_s = timeit(lambda: run(0, N)), timeit(sliced)
    print('%-34s dispatch %.3f ms %4.0f TF/s | 128-slices %.3f ms %4.0f TF/s | x%.2f' % (
        name, ms_d, flops / ms_d / 1e9, ms_s, flops / ms_s / 1e9, ms_s / ms_d))


def wide_conv(F, H, Cin, N, stride=1, residual=False):
    x = torch.randn(F, H, H, Cin, device=dev).bfloat16()
    wp = _pack_conv(torch.randn(N, Cin, 3, 3, device=dev) * 0.05)
    b = torch.zeros(N, device=dev)
    Ho = H // stride
    res = torch.randn(F, Ho, Ho, N, device=dev).bfloat16() if residual else None
    out = torch.empty(F, Ho, Ho, N, device=dev, dtype=torch.bfloat16)
    wide_case('conv F%d %d^2 %d->%d s%d res=%d' % (F, H, Cin, N, stride, residual), 2.0 * F * Ho * Ho * N * 9 * Cin,
              lambda n0, n1: ops.conv(x, wp[n0:n1], n1 - n0, out[..., n0:n1], stride=stride, bias=b[n0:n1],
                                      residual=res[..., n0:n1] if residual else None), N)


def wide_up2x(F, H, C):
    x = torch.randn(F, H, H, C, device=dev).bfloat16()
    w = torch.randn(C, C, 3, 3, device=dev) * 0.05
    b = torch.zeros(C, device=dev)
    out = torch.empty(F, 2 * H, 2 * H, C, device=dev, dtype=torch.bfloat16)
    packs = {}

    def run(n0, n1):
        if (n0, n1) not in packs:
            packs[(n0, n1)] = _pack_up2x(w[n0:n1])
        lib = ops.L.load()
        ep = ops.make_epilogue(out[..., n0:n1], b[n0:n1])
        wp4 = packs[(n0, n1)]
        ops.L.check(lib.pgt_conv_up2x_bf16(ops._p(x), F, H, H, C, x.stride(2), ops._p(wp4), wp4.stride(1), n1 - n0,
                                           ops.ctypes.byref(ep), ops._stream()))
    wide_case('up2x F%d %d^2->%d^2 %d->%d' % (F, H, 2 * H, C, C), 2.0 * F * 4 * H * H * C * 4 * C, run, C)


def halo_case(name, flops, fn):
    ms = timeit(fn)
    print('%-40s %8.3f ms %5.0f TF/s' % (name, ms, flops / ms / 1e9))


def halo_conv(F, H, Cin, N, residual=False):
    x = torch.randn(F, H, H, Cin, device=dev).bfloat16()
    wp = _pack_conv(torch.randn(N, Cin, 3, 3, device=dev) * 0.05)
    b = torch.zeros(N, device=dev)
    res = torch.randn(F, H, H, N, device=dev).bfloat16() if residual else None
    out = torch.empty(F, H, H, N, device=dev, dtype=torch.bfloat16)
    halo_case('conv F%d %d^2 %d->%d res=%d' % (F, H, Cin, N, residual), 2.0 * F * H * H * N * 9 * Cin,
              lambda: ops.conv(x, wp, N, out, bias=b, residual=res))
    del x, res, out


def halo_up2x(F, H, C):
    x = torch.randn(F, H, H, C, device=dev).bfloat16()
    wp4 = _pack_up2x(torch.randn(C, C, 3, 3, device=dev) * 0.05)
    b = torch.zeros(C, device=dev)
    out = torch.empty(F, 2 * H, 2 * H, C, device=dev, dtype=torch.bfloat16)
    halo_case('up2x F%d %d^2->%d^2 %d->%d' % (F, H, 2 * H, C, C), 2.0 * F * 4 * H * H * C * 4 * C,
              lambda: ops.conv_up2x(x, wp4, C, out, bias=b))
    del x, out


if len(sys.argv) > 1 and sys.argv[1] == 'halo':
    # the flagship workload's Cout <= 128 halo shapes at 16 clips = 48 frames (288 channels: the SFT concat buffer)
    halo_conv(48, 512, 64, 64)
    halo_conv(48, 512, 64, 64, residual=True)
    halo_conv(48, 512, 128, 64)
    halo_conv(48, 256, 64, 128)
    halo_conv(48, 256, 128, 128, residual=True)
    halo_conv(48, 256, 288, 128)
    halo_conv(48, 256, 256, 128)
    halo_up2x(48, 256, 128)
    halo_conv(48, 128, 64, 64)
    sys.exit(0)

if len(sys.argv) > 1 and sys.argv[1] == 'wide':
    wide_conv(48, 128, 256, 256)
    wide_conv(48, 128, 256, 256, residual=True)
    wide_conv(48, 128, 544, 256)
    wide_up2x(48, 128, 256)
    wide_conv(48, 32, 512, 512)
    wide_conv(48, 32, 512, 512, residual=True)
    wide_conv(48, 64, 256, 256)
    wide_conv(48, 128, 256, 256, stride=2)
    sys.exit(0)

for args in [(12, 512, 64, 64, False), (12, 512, 64, 64, True), (12, 512, 128, 64, False), (12, 256, 128, 128, False),
             (12, 256, 128, 128, True), (12, 128, 256, 256, True), (12, 128, 256, 256, False)]:
    conv_case(*args)
