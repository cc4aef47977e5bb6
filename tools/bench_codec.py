"""Times the stage-I codec kernels and methods on one GPU with CUDA events: soft_codes (soft_codes.cu) at T = 49152 and
98304 tokens (16 clips of 512^2, 8 clips of 1024^2; K = 1024 codes, E = 512), the sampler (codebook.cu), and
TDCRQVAE3.encode / decode_code at 16 clips of 512^2, on the synthetic checkpoint.  Prints one JSON line with the card
name and power limit read in the same run.

    python tools/bench_codec.py [--iters 20] [--warmup 3] [--out FILE]

Rates: soft_codes is counted as 2 T K E algorithmic FLOP (one fp32-equivalent GEMM; the kernel issues three TF32
products per term) and T K 4 bytes written + T E 4 bytes read (the minimum traffic; the in-place normalisation pass
reads and writes the output once more)."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


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
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_codec needs a CUDA device')
    import yaml
    from archs.pgtformer_arch import PGTFormer
    from pgtformer_b200 import ops
    with open(os.path.join(ROOT, 'options', 'release_test_stage_IIII_dont_need_align_version.yml')) as f:
        opt = yaml.safe_load(f)['network_g']
    opt.pop('type')
    model = PGTFormer(**opt).to('cuda')
    model.eval()
    eng = model.engine()
    cb = eng.w['codebook']
    K, E = 1024, 512
    norm = ops.codebook_pack(cb, K)[1]
    res = {'card': card(), 'iters': args.iters, 'warmup': args.warmup}
    g = torch.Generator(device='cuda').manual_seed(0)
    for T, label in ((49152, '16x512^2'), (98304, '8x1024^2')):
        z = torch.randn(T, E, device='cuda', generator=g) * 0.2
        p = torch.empty(T, K, device='cuda')
        ms = time_ms(lambda: ops.soft_codes(z, cb, norm, K, 1.0, p), args.iters, args.warmup)
        res['soft_codes_T%d' % T] = {'shape': label, 'ms': round(ms, 4),
                                     'tflops': round(2.0 * T * K * E / ms / 1e9, 1),
                                     'gbps': round((T * K * 4 + T * E * 4) / ms / 1e6, 1)}
        seed = torch.tensor([1, 2], dtype=torch.int64, device='cuda')
        idx = torch.empty(T, dtype=torch.int64, device='cuda')
        ms = time_ms(lambda: ops.sample_codes(p, seed, idx), args.iters, args.warmup)
        res['sample_codes_T%d' % T] = {'ms': round(ms, 4), 'gbps': round(T * K * 4 / ms / 1e6, 1)}
        del z, p
    x = torch.rand(48, 3, 512, 512, device='cuda', generator=g)
    code = torch.randint(0, K, (48, 32, 32, 1), device='cuda', generator=g)
    iters = max(1, args.iters // 4)
    res['encode_16x512^2_ms'] = round(time_ms(lambda: model.encode(x), iters, args.warmup), 2)
    res['decode_code_16x512^2_ms'] = round(time_ms(lambda: model.decode_code(code), iters, args.warmup), 2)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
