"""Micro-benchmark of the short-K token linears (M = 49152 rows: the 32^2-level Swin blocks and the global transformer):
CUDA events, warm (operands left in L2 by the previous repetition, as in the model) and cold (L2 flushed) timings."""
import os
import sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pgtformer_b200 import ops  # noqa: E402

dev = 'cuda'
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def timeit(fn, reps=20, cold=False):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    tot = 0.0
    for _ in range(reps):
        if cold:
            flush.zero_()
        e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
    return tot / reps


def case(M, N, K, res, act=0):
    a = torch.randn(M, K, device=dev).bfloat16()
    w = (torch.randn(N, K, device=dev) * 0.05).bfloat16()
    b = torch.zeros(N, device=dev)
    dt = torch.float32 if res == 'f32' else torch.bfloat16
    r = torch.randn(M, N, device=dev).to(dt) if res != 'none' else None
    out = torch.empty(M, N, device=dev, dtype=dt)
    fn = lambda: ops.linear(a, w, out, bias=b, residual=r, act=act)
    w_ms, c_ms = timeit(fn), timeit(fn, cold=True)
    fl = 2.0 * M * N * K
    by = M * K * 2 + M * N * (2 if dt == torch.bfloat16 else 4) * (2 if r is not None else 1) + N * K * 2
    print('linear M%d N%d K%d res=%-4s act=%d: warm %.1f us %.0f TF/s %.2f TB/s | cold %.1f us %.0f TF/s %.2f TB/s' % (
        M, N, K, res, act, w_ms * 1e3, fl / w_ms / 1e9, by / w_ms / 1e9, c_ms * 1e3, fl / c_ms / 1e9, by / c_ms / 1e9))


def wide(M, N, K, res):
    """The launch dispatch_gemm picks against the same product launched as 128-column slices (the 128-wide kernel)."""
    a = torch.randn(M, K, device=dev).bfloat16()
    w = (torch.randn(N, K, device=dev) * 0.05).bfloat16()
    b = torch.zeros(N, device=dev)
    dt = torch.float32 if res == 'f32' else torch.bfloat16
    r = torch.randn(M, N, device=dev).to(dt) if res != 'none' else None
    out = torch.empty(M, N, device=dev, dtype=dt)
    run = lambda n0, n1: ops.linear(a, w[n0:n1], out[:, n0:n1], bias=b[n0:n1],
                                    residual=r[:, n0:n1] if r is not None else None)

    def sliced():
        for n0 in range(0, N, 128):
            run(n0, min(N, n0 + 128))
    ms_d, ms_s = timeit(lambda: run(0, N)), timeit(sliced)
    fl = 2.0 * M * N * K
    print('linear M%d N%d K%d res=%-4s dispatch %.1f us %4.0f TF/s | 128-slices %.1f us %4.0f TF/s | x%.2f' % (
        M, N, K, res, ms_d * 1e3, fl / ms_d / 1e9, ms_s * 1e3, fl / ms_s / 1e9, ms_s / ms_d))


if len(sys.argv) > 1 and sys.argv[1] == 'wide':
    for N, K, res in [(1024, 512, 'none'), (512, 1024, 'none'), (512, 1024, 'f32'), (512, 512, 'none'),
                      (512, 512, 'bf16'), (512, 512, 'f32'), (1536, 512, 'none'), (768, 256, 'none')]:
        wide(49152, N, K, res)
    sys.exit(0)

M = int(sys.argv[1]) if len(sys.argv) > 1 else 49152
for N, K, res, act in [(512, 512, 'none', 0), (512, 512, 'bf16', 0), (512, 512, 'f32', 0), (1024, 512, 'none', 0),
                       (1024, 512, 'none', 1), (1536, 512, 'none', 0), (512, 1024, 'f32', 0), (512, 1024, 'bf16', 0)]:
    case(M, N, K, res, act)
