"""Times the d = 64 global attention (`pgt_mha_fwd` -> mha_tc_kernel) and the fp32-input LayerNorm of the global
transformer at the workload's shapes on one GPU with CUDA events:

- mha: 16 clips x L = 3072 x 8 heads (16 clips of 512^2) and 8 x 12288 x 8 (8 clips of 1024^2), d = 64;
- layernorm: fp32 x [49152, 512] -> bf16, with the positional second output (norm1) and without (norm2).

With `--baseline-lib` (a libpgt_b200.so built from another commit) both libraries are timed in one run, alternating
round by round on the same inputs, and their outputs are compared.  Prints one JSON line with the card name, power
limit and maximum SM clock read in the same run.

    python tools/bench_mha.py [--baseline-lib PATH] [--rounds 5] [--iters 20] [--out FILE]"""
import argparse
import ctypes
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from bench_codec import card, time_ms  # noqa: E402


def open_lib(path):
    from pgtformer_b200 import _lib
    if path is None:
        return _lib.load()
    lib = ctypes.CDLL(os.path.abspath(path))
    for name in ('pgt_mha_fwd', 'pgt_layernorm'):
        res, args = _lib.SIGNATURES[name]
        getattr(lib, name).restype = res
        getattr(lib, name).argtypes = args
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--baseline-lib', default=None)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_mha needs a CUDA device')
    from pgtformer_b200 import _lib
    libs = {'this': open_lib(None)}
    if args.baseline_lib:
        libs['baseline'] = open_lib(args.baseline_lib)
    dev = 'cuda'
    g = torch.Generator().manual_seed(0)
    P = lambda t: ctypes.c_void_p(t.data_ptr())
    st = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    cases = {}
    for clips, L in ((16, 3072), (8, 12288)):
        T, E = clips * L, 512
        q, k, v = (torch.randn(T, E, generator=g).to(torch.bfloat16).to(dev) for _ in range(3))
        outs = {n: torch.empty(T, E, dtype=torch.bfloat16, device=dev) for n in libs}

        def mha(lib, out, q=q, k=k, v=v, clips=clips, L=L):
            _lib.check(lib.pgt_mha_fwd(P(q), 512, P(k), 512, P(v), 512, clips, L, 8, 64, P(out), 512, st()))
        cases['mha_%dx%d' % (clips, L)] = (mha, outs, 4.0 * clips * 8 * L * L * 64)
    T, C = 49152, 512
    x = (torch.randn(T, C, generator=g) * 3 + 0.5).to(dev)
    gam, bet = (1 + 0.1 * torch.randn(C, generator=g)).to(dev), (0.1 * torch.randn(C, generator=g)).to(dev)
    pos = torch.randn(T, C, generator=g).to(torch.bfloat16).to(dev)
    for with_pos in (True, False):
        outs = {n: torch.empty(2 if with_pos else 1, T, C, dtype=torch.bfloat16, device=dev) for n in libs}

        def ln(lib, out, with_pos=with_pos):
            _lib.check(lib.pgt_layernorm(P(x), C, _lib.F32, T, C, P(gam), P(bet), 1e-5, P(out[0]), C,
                                         P(pos) if with_pos else None, C if with_pos else 0,
                                         P(out[1]) if with_pos else None, C if with_pos else 0, st()))
        cases['layernorm_f32_%dx%d%s' % (T, C, '_pos' if with_pos else '')] = (ln, outs, None)

    res = {'card': card(), 'rounds': args.rounds, 'iters': args.iters, 'ms': {}, 'ms_all': {}}
    for name, (fn, outs, flops) in cases.items():
        t = {n: [] for n in libs}
        for n, lib in libs.items():                     # warm up every library on every shape
            time_ms(lambda: fn(lib, outs[n]), 2, 2)
        for _ in range(args.rounds):
            for n, lib in libs.items():
                t[n].append(time_ms(lambda: fn(lib, outs[n]), args.iters, 1))
        res['ms'][name] = {n: min(v) for n, v in t.items()}
        res['ms_all'][name] = t
        if flops is not None:
            res.setdefault('tflops', {})[name] = {n: flops / (min(v) * 1e-3) / 1e12 for n, v in t.items()}
        if 'baseline' in libs:
            a, b = outs['this'].float(), outs['baseline'].float()
            res.setdefault('bit_identical', {})[name] = bool(torch.equal(outs['this'], outs['baseline']))
            res.setdefault('max_abs_diff', {})[name] = (a - b).abs().max().item()
    line = json.dumps(res)
    print(line, flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
