"""Times CodeFormer.forward (w = 0.5, adain on) and VQAutoEncoder.forward on one GPU: images/s at b = 1 and b = 16 of
512^2 from CUDA events after warm-up (synthetic checkpoint, default constructor arguments, inputs in [-1, 1]), the
achieved TFLOP/s over the FLOPs counted from the shapes (model_flops), and one profiled forward per model split into
conv + linear GEMMs (the GEMM / conv kernel class minus the transformer's share: the 3x3 convs, and also the AttnBlocks'
q | k | v and proj_out projections, the 1x1 shortcuts and the fusion blocks' convs), AttnBlock cores (the mha class
minus the transformer's share), the 9-layer transformer (profiled on its own, CodeFormer only) and the rest.  The profiled split
puts CUDA events around every launch (pgt_profile_begin / end), so its sum is above the unprofiled time.  Prints one
JSON line with the card's name and power limit read in the same run.

    python tools/bench_codeformer.py [--iters 5] [--warmup 2] [--out FILE]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from bench_tdrqvae import card  # noqa: E402


def model_flops(arch, H, W, codeformer, w=0.5):
    """Multiply-adds x 2 of one image's forward, counted from the block list: convs, AttnBlocks (1x1 projections and
    the two L x L products), and for CodeFormer the transformer, feat_emb / idx_pred and the fusion blocks."""
    def conv(h, w_, cin, cout, k):
        return 2.0 * h * w_ * cin * cout * k * k

    def res(h, w_, cin, cout):
        return conv(h, w_, cin, cout, 3) + conv(h, w_, cout, cout, 3) + (conv(h, w_, cin, cout, 1) if cin != cout else 0)

    def blocks(bl, scale):
        f = 0.0
        for kind, cin, cout, r in bl:
            h, w_ = r * H // (arch.img_size * scale), r * W // (arch.img_size * scale)
            if kind in ('conv_in', 'conv_out'):
                f += conv(h, w_, cin, cout, 3)
            elif kind == 'res':
                f += res(h, w_, cin, cout)
            elif kind == 'attn':
                L = h * w_
                f += 4 * conv(h, w_, cin, cin, 1) + 4.0 * L * L * cin
            elif kind == 'down':
                f += conv(h // 2, w_ // 2, cin, cin, 3)
            elif kind == 'up':
                f += conv(2 * h, 2 * w_, cin, cin, 3)
        return f
    f = blocks(arch.enc_blocks, 1) + blocks(arch.gen_blocks, 1)
    if not codeformer:
        return f
    L, E, D = H * W // arch.down ** 2, arch.embed_dim, arch.dim_embd
    f += 2.0 * L * E * D + arch.n_layers * (2.0 * L * D * 3 * D + 4.0 * L * L * D + 2.0 * L * D * D + 8.0 * L * D * D)
    f += 2.0 * L * D * arch.n_embed
    if w > 0:
        from pgtformer_b200.spec import CODEFORMER_CHANNELS
        for key in arch.connect_list:
            c, s = CODEFORMER_CHANNELS[key], int(key)
            f += res(s, s, 2 * c, c) + 4 * conv(s, s, c, c, 3)
    return f


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def profiled(fn):
    from pgtformer_b200 import ops
    fn()
    torch.cuda.synchronize()
    ops.profile_begin()
    fn()
    torch.cuda.synchronize()
    return ops.profile_end()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out')
    args = ap.parse_args()
    from archs import CodeFormer, VQAutoEncoder
    res = {'card': card()}
    with torch.no_grad():
        for name, cls in (('codeformer', CodeFormer), ('vqgan', VQAutoEncoder)):
            m = cls().to('cuda').eval()
            cfm = name == 'codeformer'
            fwd = (lambda x: m(x, w=0.5, adain=True)) if cfm else (lambda x: m(x))
            for b in (1, 16):
                x = (torch.rand(b, 3, 512, 512, generator=torch.Generator().manual_seed(b)) * 2 - 1).to('cuda')
                ms = timed(lambda: fwd(x), args.iters, args.warmup)
                fl = b * model_flops(m.arch, 512, 512, cfm)
                r = {'ms': round(ms, 3), 'images_per_s': round(1e3 * b / ms, 2), 'gflop': round(fl / 1e9, 1),
                     'tflops': round(fl / ms / 1e9, 1)}
                if b == 16:
                    prof = profiled(lambda: fwd(x))
                    tr = {}
                    if cfm:
                        eng = m.engine()
                        lq = torch.randn(b * 256, 256, generator=torch.Generator().manual_seed(3)).to('cuda').bfloat16()
                        tr = profiled(lambda: eng.global_transformer(lq, eng.pos(b), b))
                    ms_of = lambda p, k: p.get(k, (0, 0.0, 0))[1]
                    total = sum(v[1] for v in prof.values())
                    t_tr = sum(v[1] for v in tr.values())
                    convs = ms_of(prof, 'gemm_tc') - ms_of(tr, 'gemm_tc')
                    attn = ms_of(prof, 'mha') - ms_of(tr, 'mha')
                    r['profiled_ms'] = {'conv_linear_gemms': round(convs, 2), 'attn_block_cores': round(attn, 2),
                                        'transformer': round(t_tr, 2), 'rest': round(total - convs - attn - t_tr, 2),
                                        'total': round(total, 2)}
                res['%s_b%d' % (name, b)] = r
            del m
            torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
