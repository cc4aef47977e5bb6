"""RQVAE on one GPU.  (1) The exact L2 argmin, split over code ranges (l2_argmin_tc_split with the default choice of
ranges, ops.argmin_splits) against the unsplit sweep (l2_argmin_tc), D = 4 depths back to back, at T in {64, 1024, 4096}
tokens, K in {2048, 16384} codes, E = 256.  (2) forward, get_codes and decode_code of the R1 configuration
(oracle/make_rqvae_golden.py: ch 128, f = 32, a shared 2048-code codebook of depth 4) on 256^2 images at b in
{1, 16, 64}, synthetic weights.  CUDA events around `iters` calls after `warmup` calls of the same shape; every
measurement is repeated over `rounds` rounds, the two argmins alternating within each round.  One JSON line per
measurement, plus the card.

    python tools/bench_rqvae.py [--iters 20] [--warmup 3] [--rounds 2] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BATCHES = (1, 16, 64)
ARGMIN_T = (64, 1024, 4096)
ARGMIN_K = (2048, 16384)


def card():
    info = {'name': torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=30)
        info['power_limit_clocks_max_sm'] = r.stdout.strip()
    except Exception as e:                                   # the timing stays valid; the record says why it is missing
        info['power_limit_clocks_max_sm'] = 'unavailable: %s' % e
    return info


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    from archs.rqvae_arch import RQVAE
    from oracle.make_rqvae_golden import R1
    from pgtformer_b200 import ops
    rows = [dict(card(), config='R1')]
    E, D = 256, 4
    for K in ARGMIN_K:
        g = torch.Generator().manual_seed(K)
        cb = torch.randn(K + 1, E, generator=g).cuda()
        pack = ops.codebook_pack(cb, K)
        for T in ARGMIN_T:
            z = torch.randn(T, E, generator=g).cuda()
            a, b = (torch.empty(T, dtype=torch.int64, device='cuda') for _ in range(2))
            S = ops.argmin_splits(T, K)
            fns = {'unsplit': lambda: [ops.l2_argmin_tc(z, cb, pack, K, a) for _ in range(D)],
                   'split': lambda: [ops.l2_argmin_tc_split(z, cb, pack, K, b, splits=S) for _ in range(D)]}
            for r in range(args.rounds):
                for name, fn in fns.items():
                    ms = time_ms(fn, args.iters, args.warmup)
                    rows.append({'argmin': name, 'T': T, 'K': K, 'E': E, 'D': D, 'splits': S if name == 'split' else 1,
                                 'round': r, 'ms': round(ms, 4)})
                    print(json.dumps(rows[-1]), flush=True)
            assert torch.equal(a, b)
    g = dict(R1)
    g.pop('type')
    m = RQVAE(**g).cuda().eval()
    for r in range(args.rounds):
        for b in BATCHES:
            x = torch.rand(b, 3, 256, 256, generator=torch.Generator().manual_seed(b)).cuda()
            code = m.get_codes(x)
            for name, fn in (('forward', lambda: m(x)), ('get_codes', lambda: m.get_codes(x)),
                             ('decode_code', lambda: m.decode_code(code))):
                ms = time_ms(fn, args.iters, args.warmup)
                rows.append({'method': name, 'b': b, 'round': r, 'ms': round(ms, 3),
                             'images_per_s': round(1e3 * b / ms, 1)})
                print(json.dumps(rows[-1]), flush=True)
    print(json.dumps(rows[0]))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
