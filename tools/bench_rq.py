"""Times the residual quantiser at depth D on one GPU with CUDA events, configurations alternated within the run:

- the quantiser alone (Engine.quantize: per depth l2_argmin_tc + rq_residual) at T = 49152 tokens (16 clips of 512^2),
  K = 1024, E = 512, D in {1, 2, 4}, shared and separate codebooks;
- TDCRQVAE3.forward at 16 clips of 512^2, D = 1 against D = 4 (separate codebooks);
- PGTFormer.forward (CUDA-graph replay) at 16 clips of 512^2, D = 1 against D = 2 (shared, as in the options files).

Synthetic checkpoints (seed 0).  Prints one JSON line with the card name and power limit read in the same run.

    python tools/bench_rq.py [--rounds 3] [--iters 5] [--out FILE]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from bench_codec import card, time_ms  # noqa: E402


def network_g(depth, shared):
    import yaml
    with open(os.path.join(ROOT, 'options', 'release_test_stage_IIII_dont_need_align_version.yml')) as f:
        g = yaml.safe_load(f)['network_g']
    g.pop('type')
    g['code_shape'] = [32, 32, depth]
    g['shared_codebook'] = shared
    return g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_rq needs a CUDA device')
    from archs.pgtformer_arch import PGTFormer
    dev = 'cuda'
    res = {'card': card(), 'rounds': args.rounds, 'iters': args.iters}
    # ---- quantiser alone: one engine per configuration, the same z for all
    T, E = 49152, 512
    z = torch.randn(T, E, generator=torch.Generator().manual_seed(1)).mul_(0.5).to(dev)
    quant = {}
    for D in (1, 2, 4):
        for shared in ((True,) if D == 1 else (True, False)):
            eng = PGTFormer(**network_g(D, shared)).to(dev).engine()
            eng.quantize(z)
            quant['D%d_%s' % (D, 'shared' if shared else 'separate')] = eng
    times = {k: [] for k in quant}
    for _ in range(args.rounds):
        for k, eng in quant.items():
            times[k].append(time_ms(lambda: eng.quantize(z), args.iters * 4, 2))
    res['quantize_ms'] = {k: min(v) for k, v in times.items()}
    res['quantize_ms_all'] = times
    del quant
    # ---- whole models at 16 clips of 512^2
    x = torch.rand(48, 3, 512, 512, generator=torch.Generator().manual_seed(2)).to(dev)
    for label, cfgs, call in (('tdcrqvae3_forward_ms', ((1, True), (4, False)), lambda m: m.forward_vq(x)),
                              ('pgtformer_forward_graphed_ms', ((1, True), (2, True)), lambda m: m(x, w=1.0))):
        models = {}
        for D, shared in cfgs:
            m = PGTFormer(**network_g(D, shared)).to(dev)
            m.eval()
            m.cuda_graph = label.startswith('pgtformer')
            call(m)
            models['D%d' % D] = m
        t = {k: [] for k in models}
        for _ in range(args.rounds):
            for k, m in models.items():
                t[k].append(time_ms(lambda: call(m), args.iters, 1))
        res[label] = {k: min(v) for k, v in t.items()}
        res[label + '_all'] = t
        del models
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line, flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
