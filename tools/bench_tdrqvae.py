"""Times the wide-head attention core (attn_wide_tc.cu, `pgt_mha_fwd` with d = 256 / 512: TDRQVAE's dense AttnBlock
core) on one GPU with CUDA events, over 48 frames at the (d, L) of the AttnBlock levels of 512^2 and 1024^2 clips:
(256, 16384) and (256, 4096) are the 128^2 and 64^2 levels, (512, 1024) and (512, 4096) the 32^2 level and mid blocks.
Rates count 4 F L^2 d FLOP (the two products).  torch's scaled_dot_product_attention on the same bf16 tensors goes
beside it as a yardstick at d = 256 (its flash backend stops at 256).  Prints one JSON line with the card's name,
power limit and max SM clock read in the same run.

    python tools/bench_tdrqvae.py [--iters 10] [--warmup 2] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FRAMES = 48
SHAPES = ((256, 16384), (256, 4096), (512, 1024), (512, 4096))


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
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_tdrqvae needs a CUDA device')
    import torch.nn.functional as F
    from pgtformer_b200 import ops
    res = {'card': card(), 'iters': args.iters, 'warmup': args.warmup, 'frames': FRAMES}
    g = torch.Generator(device='cuda').manual_seed(0)
    for d, L in SHAPES:
        T = FRAMES * L
        qkv = (torch.randn(T, 3 * d, device='cuda', generator=g) * 1.5).to(torch.bfloat16)
        q, k, v = qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:]
        out = torch.empty(T, d, dtype=torch.bfloat16, device='cuda')
        flop = 4.0 * FRAMES * L * L * d
        ms = time_ms(lambda: ops.mha(q, k, v, FRAMES, L, 1, d, out), args.iters, args.warmup)
        rec = {'ms': round(ms, 3), 'tflops': round(flop / ms / 1e9, 1)}
        if d == 256:
            qs, ks, vs = (t.reshape(FRAMES, 1, L, d) for t in (q, k, v))
            ms = time_ms(lambda: F.scaled_dot_product_attention(qs, ks, vs), args.iters, args.warmup)
            rec['sdpa_ms'] = round(ms, 3)
            rec['sdpa_tflops'] = round(flop / ms / 1e9, 1)
        res['core_d%d_L%d' % (d, L)] = rec
        del qkv, out
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
