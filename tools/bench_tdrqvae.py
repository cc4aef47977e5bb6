"""Times the wide-head attention core (attn_wide_tc.cu, `pgt_mha_fwd` with d = 256 / 512: TDRQVAE's dense AttnBlock
core) on one GPU with CUDA events, over 48 frames at the (d, L) of the AttnBlock levels of 512^2 and 1024^2 clips:
(256, 16384) and (256, 4096) are the 128^2 and 64^2 levels, (512, 1024) and (512, 4096) the 32^2 level and mid blocks.
Rates count 4 F L^2 d FLOP (the two products).  torch's scaled_dot_product_attention on the same bf16 tensors goes
beside it as a yardstick at d = 256 (its flash backend stops at 256).  Prints one JSON line with the card's name,
power limit and max SM clock read in the same run.

--model times the whole registered TDRQVAE.forward (synthetic checkpoint, this repo's network_g with type TDRQVAE) on
16 clips x 3 frames of 512^2 and on 7 clips x 7 frames of 512^2 instead: ms per forward and frames/s from CUDA events
after warm-up, the algorithmic FLOPs counted from the shapes (model_flops), and one profiled forward split per kernel
class (pgt_profile_begin / end, CUDA events around every launch, as tools/layer_profile.py): the AttnBlock cores (mha),
GEMMs and convs (gemm_tc), the Video-Swin window attention (window3d) and the rest.

    python tools/bench_tdrqvae.py [--iters 10] [--warmup 2] [--out FILE]
    python tools/bench_tdrqvae.py --model [--iters 3] [--warmup 1] [--out FILE]
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


MODEL_CASES = ((16, 3), (7, 7))           # (clips, frames per clip) at 512^2


def model_flops(a, b, t, H, W):
    """Algorithmic FLOPs (2 per multiply-add) of one TDRQVAE.forward on b clips of t frames of H x W, counted from the
    shapes: every conv / linear, the AttnBlock cores (4 L^2 C: q k^T and P v), the Video-Swin window cores (4 N C per
    token, N the tokens of a clipped window; padded tokens not counted) and the L2 argmin.  Returns {class: FLOPs}."""
    F_ = b * t
    fl = {'attn_core': 0.0, 'gemm_conv': 0.0, 'window3d': 0.0, 'argmin': 0.0}

    def conv(hw, cin, cout, k=3):
        fl['gemm_conv'] += 2.0 * F_ * hw * cin * cout * k * k

    def res(hw, cin, cout):
        conv(hw, cin, cout)
        conv(hw, cout, cout)
        if cin != cout:
            conv(hw, cin, cout, 1)

    def attn(hw, c):
        conv(hw, c, 3 * c, 1)
        conv(hw, c, c, 1)
        fl['attn_core'] += 4.0 * F_ * hw * hw * c

    hh, ww = H // a.down, W // a.down
    E, T = a.embed_dim, F_ * hh * ww
    ws = [min(s, w) for s, w in zip((t, hh, ww), a.window_size)]

    def swin():
        fl['gemm_conv'] += a.stages_atten * 2.0 * T * (3 * E * E + E * E + 8 * E * E)
        fl['window3d'] += a.stages_atten * 4.0 * T * ws[0] * ws[1] * ws[2] * E

    hw, cin = H * W, a.ch
    conv(hw, 3, a.ch)
    for lvl in range(a.num_levels):
        for _ in range(a.num_res_blocks):
            res(hw, cin, a.level_ch[lvl])
            cin = a.level_ch[lvl]
            if a.level_has_attn[lvl]:
                attn(hw, cin)
        if lvl != a.num_levels - 1:
            hw //= 4
            conv(hw, cin, cin)
    res(hw, cin, cin), attn(hw, cin), res(hw, cin, cin)
    conv(hw, cin, a.z_channels)
    conv(hw, a.z_channels, E, 1)
    swin()
    fl['argmin'] += 2.0 * T * a.n_embed * E
    swin()
    conv(hw, E, a.z_channels, 1)
    conv(hw, a.z_channels, cin)
    res(hw, cin, cin), attn(hw, cin), res(hw, cin, cin)
    for lvl in reversed(range(a.num_levels)):
        for _ in range(a.num_res_blocks + 1):
            res(hw, cin, a.level_ch[lvl])
            cin = a.level_ch[lvl]
            if a.level_has_attn[lvl]:
                attn(hw, cin)
        if lvl != 0:
            hw *= 4
            conv(hw, cin, cin)
    conv(hw, cin, a.out_ch)
    return fl


def bench_model(args, res):
    import yaml
    from archs.tdrqvae_arch import TDRQVAE
    from pgtformer_b200 import ops
    with open(os.path.join(ROOT, 'options', 'release_test_stage_IIII_dont_need_align_version.yml')) as f:
        g = yaml.safe_load(f)['network_g']
    g['type'] = 'TDRQVAE'
    model = TDRQVAE(**g).cuda().eval()
    H = W = 512
    for b, t in MODEL_CASES:
        x = torch.rand(b, t, 3, H, W, device='cuda', generator=torch.Generator(device='cuda').manual_seed(b * t))
        ms = time_ms(lambda: model(x), args.iters, args.warmup)
        fl = model_flops(model.arch, b, t, H, W)
        total = sum(fl.values())
        ops.profile_begin()
        model(x)
        prof = ops.profile_end()
        split = {'attn_core': prof['mha'][1], 'gemm_conv': prof['gemm_tc'][1], 'window3d': prof['window_attn'][1]}
        split['rest'] = sum(v[1] for k, v in prof.items() if k not in ('mha', 'gemm_tc', 'window_attn'))
        res['model_b%d_t%d_%d' % (b, t, H)] = {
            'frames': b * t, 'ms_per_forward': round(ms, 2), 'frames_per_s': round(1e3 * b * t / ms, 1),
            'gflop': {k: round(v / 1e9, 1) for k, v in fl.items()}, 'tflops': round(total / ms / 1e9, 1),
            'profiled_ms': {k: round(v, 2) for k, v in split.items()},
            'profiled_launches': sum(v[2] for v in prof.values())}
        del x
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=None)
    ap.add_argument('--warmup', type=int, default=None)
    ap.add_argument('--model', action='store_true', help='time the whole TDRQVAE.forward instead of the cores')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_tdrqvae needs a CUDA device')
    if args.iters is None:
        args.iters = 3 if args.model else 10
    if args.warmup is None:
        args.warmup = 1 if args.model else 2
    if args.model:
        res = {'card': card(), 'iters': args.iters, 'warmup': args.warmup, 'size': 512}
        bench_model(args, res)
        line = json.dumps(res)
        print(line)
        if args.out:
            with open(args.out, 'w') as f:
                f.write(line + '\n')
        return
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
