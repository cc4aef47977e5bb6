"""Eager calls against CUDA-graph replay (model.cuda_graph = True) of the five models whose calls replay: CodeFormer
(forward, w = 0.5, adain on) and VQAutoEncoder forward on 512^2 images, RQVAE R1 forward / get_codes / decode_code on
256^2 images (oracle/make_rqvae_golden.py), TDRQVAE forward and TDCRQVAE3 forward on 3-frame clips of 512^2, at b = 1, 4
and 16 images (clips for the two video models), synthetic checkpoints.

For every (model, call, b): both modes warmed up (the graph captured) and checked bit for bit against each other, then
`rounds` rounds, each timing `iters` eager calls and `iters` graphed calls back to back with CUDA events, so that the
two modes alternate within the run.  Reports ms per call for each round, calls/s and images/s (frames/s for the video
models) of the median round, the kernel launches of one eager call (ops.launch_count) and, at b = 1, the summed kernel
time of one profiled eager call (ops.profile_begin / end: CUDA events around every launch, in a separate pass), the part
of the eager call the GPU is busy.  Prints one JSON line with the card's name and power limit read in the same run.

    python tools/bench_graphs.py [--iters N] [--rounds 3] [--warmup 2] [--models codeformer,vqgan,...] [--out FILE]

--iters defaults to 64 / b calls per timed window (at least 4)."""
import argparse
import copy
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from bench_tdrqvae import card  # noqa: E402

BATCHES = (1, 4, 16)
MODELS = ('codeformer', 'vqgan', 'rqvae_r1', 'tdrqvae', 'tdcrqvae3')


def _network_g():
    import yaml
    with open(os.path.join(ROOT, 'options', 'release_test_stage_IIII_dont_need_align_version.yml')) as f:
        return yaml.safe_load(f)['network_g']


def build(name):
    """-> (model, {call: (fn(inputs), make_inputs(b))}, frames per b)."""
    from archs import CodeFormer, VQAutoEncoder
    from archs.pgtformer_arch import TDCRQVAE3
    from archs.rqvae_arch import RQVAE
    from archs.tdrqvae_arch import TDRQVAE
    gen = lambda b: torch.Generator().manual_seed(b)
    if name in ('codeformer', 'vqgan'):
        m = (CodeFormer if name == 'codeformer' else VQAutoEncoder)().cuda().eval()
        img = lambda b: (torch.rand(b, 3, 512, 512, generator=gen(b)) * 2 - 1).cuda()
        fwd = (lambda x: m(x, w=0.5, adain=True)) if name == 'codeformer' else (lambda x: m(x))
        return m, {'forward': (fwd, img)}, 1
    if name == 'rqvae_r1':
        from oracle.make_rqvae_golden import R1
        g = copy.deepcopy(R1)
        g.pop('type')
        m = RQVAE(**g).cuda().eval()
        img = lambda b: torch.rand(b, 3, 256, 256, generator=gen(b)).cuda()

        def code(b):
            m.cuda_graph = False
            return m.get_codes(img(b)).clone()
        return m, {'forward': (lambda x: m(x), img), 'get_codes': (lambda x: m.get_codes(x), img),
                   'decode_code': (lambda c: m.decode_code(c), code)}, 1
    g = _network_g()
    if name == 'tdrqvae':
        g['type'] = 'TDRQVAE'
        m = TDRQVAE(**g).cuda().eval()
        return m, {'forward': (lambda x: m(x), lambda b: torch.rand(b, 3, 3, 512, 512, generator=gen(b)).cuda())}, 3
    g.pop('type')
    m = TDCRQVAE3(**g).cuda().eval()
    return m, {'forward': (lambda x: m(x), lambda b: torch.rand(3 * b, 3, 512, 512, generator=gen(b)).cuda())}, 3


def flat(o):
    if torch.is_tensor(o):
        return [o]
    if isinstance(o, dict):
        return [t for k in sorted(o) for t in flat(o[k])]
    if isinstance(o, (tuple, list)):
        return [t for v in o for t in flat(v)]
    return []


def window_ms(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def bench_call(m, fn, x, frames, iters, rounds, warmup, profile):
    from pgtformer_b200 import ops
    eager = [t.clone() for t in flat(fn(x))]
    m.cuda_graph = True
    graphed = flat(fn(x))                                   # warm-up and capture of this key
    same = len(graphed) == len(eager) and all(torch.equal(u, v) for u, v in zip(graphed, eager))
    for _ in range(warmup):
        fn(x)
    m.cuda_graph = False
    for _ in range(warmup):
        fn(x)
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    fn(x)
    launches = ops.launch_count() - n0
    ms = {'eager': [], 'graphed': []}
    for _ in range(rounds):
        for mode in ('eager', 'graphed'):
            m.cuda_graph = mode == 'graphed'
            ms[mode].append(round(window_ms(lambda: fn(x), iters), 3))
    m.cuda_graph = False
    r = {'iters': iters, 'bit_identical': same, 'launches_per_call': launches}
    for mode in ('eager', 'graphed'):
        med = statistics.median(ms[mode])
        r[mode] = {'ms_per_call': ms[mode], 'calls_per_s': round(1e3 / med, 1),
                   'images_per_s': round(1e3 * frames / med, 1)}
    r['speedup_median'] = round(statistics.median(ms['eager']) / statistics.median(ms['graphed']), 3)
    if profile:
        torch.cuda.synchronize()
        ops.profile_begin()
        fn(x)
        torch.cuda.synchronize()
        prof = ops.profile_end()
        r['profiled_kernel_ms'] = round(sum(v[1] for v in prof.values()), 3)
        r['profiled_launches'] = sum(v[2] for v in prof.values())
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=None)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--models', default=','.join(MODELS))
    ap.add_argument('--batches', default=','.join(str(b) for b in BATCHES))
    ap.add_argument('--out')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_graphs needs a CUDA device')
    res = {'card': card(), 'rounds': args.rounds, 'warmup': args.warmup}
    for name in args.models.split(','):
        m, calls, per = build(name)
        for call, (fn, make) in calls.items():
            for b in (int(v) for v in args.batches.split(',')):
                x = make(b)
                iters = args.iters or max(4, 64 // b)
                r = bench_call(m, fn, x, per * b, iters, args.rounds, args.warmup, profile=b == 1)
                res['%s_%s_b%d' % (name, call, b)] = r
                print(json.dumps({'case': '%s_%s_b%d' % (name, call, b), **r}), flush=True)
                del x
                m.refresh()                               # a new engine: this key's graph and its memory pool go
                torch.cuda.empty_cache()
        del m, calls, fn, make
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
