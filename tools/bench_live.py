"""Live restoration (pgtformer_b200/video.py::LiveRestorer) on a seeded synthetic video: per-frame latency and
sustained frames/s, eager and replayed from CUDA graphs, beside the batched VideoRestorer.

* latency: host clock from push(f[i+1]) to restored frame i in host memory (push returns it), p50 / p90 / p99 over
  every push that returns a frame, in every round;
* frames/s: `rounds` rounds, each streaming the whole video eagerly and then graphed (the two alternate within the
  run), frames / wall time of the stream (flush included); the median round is reported;
* VideoRestorer.restore at clips_per_batch 1 and 16 on the same frames, in the same run, for reference;
* C-ABI launches of one eager live step (ops.launch_count) and of one graphed step (none expected), and the work of the
  per-frame part of a step (frame_step) against its window part (window_step): FLOPs of the GEMM / attention kernels and
  bytes of the normalisation / gather kernels, as the C ABI's profile counters compute them from the launch shapes;
* the card's name, power limit and max SM clock, read in the same run.

Prints one JSON line.

    python tools/bench_live.py [--frames 300] [--size 512] [--rounds 3] [--w 1.0] [--weights CKPT] [--out FILE]
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from bench_tdrqvae import card  # noqa: E402

FLOP_CLASSES = ('gemm_tc', 'window_attn', 'mha', 'l2_argmin')


def build_model(weights):
    import yaml
    from archs.pgtformer_arch import PGTFormer
    with open(os.path.join(ROOT, 'options', 'release_test_stage_IIII_dont_need_align_version.yml')) as f:
        opt = yaml.safe_load(f)
    kw = dict(opt['network_g'])
    kw.pop('type')
    m = PGTFormer(**kw)
    if weights:
        sd = torch.load(weights, map_location='cpu')
        key = opt['path'].get('param_key_g') or 'params_ema'
        m.load_state_dict(sd.get(key, sd.get('params', sd)) if isinstance(sd, dict) else sd)
    m = m.cuda().eval()
    m.cuda_graph = False
    return m


def live_round(live, frames):
    """Streams frames through live; -> (seconds, [latency of every push that returned a frame], outputs)."""
    lat, outs = [], []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for f in frames:
        a = time.perf_counter()
        r = live.push(f)
        if r is not None:
            lat.append(time.perf_counter() - a)
            outs.append(r)
    outs.append(live.flush())
    return time.perf_counter() - t0, lat, outs


def pct(xs, q):
    xs = sorted(xs)
    return xs[min(len(xs) - 1, int(round(q / 100.0 * (len(xs) - 1))))]


def step_work(model, size):
    """Launches and profile counters of one eager frame_step and one eager window_step at steady state."""
    from pgtformer_b200 import ops
    from pgtformer_b200.video import LiveRestorer
    live = LiveRestorer(model, cuda_graph=False)
    f = np.random.RandomState(1).randint(0, 256, size=(4, size, size, 3), dtype=np.uint8)
    for i in range(3):
        live.push(f[i])
    sess = live._pool._state              # re-running its last step's halves rewrites the same bytes
    torch.cuda.synchronize()
    res = {}
    with torch.cuda.device(sess.eng.dev):
        for name, fn in (('frame_step', lambda: sess.run(1, 0)), ('window_step', lambda: sess.run(0, 1))):
            n = ops.launch_count()
            fn()
            torch.cuda.synchronize()
            launches = ops.launch_count() - n
            ops.profile_begin()
            fn()
            torch.cuda.synchronize()
            prof = ops.profile_end()
            res[name] = {'launches': launches,
                         'gflop': round(sum(prof[c][0] for c in FLOP_CLASSES) / 1e9, 2),
                         'mbytes': round(sum(v[0] for c, v in prof.items() if c not in FLOP_CLASSES) / 1e6, 1)}
    ring = sess.ring
    res['ring_mbytes_per_slot'] = round((ring['pos'][0].numel() * 2 + ring['h'][0].numel() * 2
                                         + sum(t[0].numel() * 2 for t in ring['feats'].values())
                                         + (ring['h_stats'][0].numel() * 4 if 'h_stats' in ring else 0)) / 1e6, 2)
    live.flush()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=300)
    ap.add_argument('--size', type=int, default=512)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--w', type=float, default=1.0)
    ap.add_argument('--weights', default=None, help='a PGTFormer checkpoint; synthetic weights without it')
    ap.add_argument('--out', default=None, help='also write the JSON line to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_live.py measures on a CUDA device; none found')
    from pgtformer_b200 import ops
    from pgtformer_b200.video import LiveRestorer, VideoRestorer
    model = build_model(args.weights)
    frames = np.random.RandomState(0).randint(0, 256, size=(args.frames, args.size, args.size, 3), dtype=np.uint8)
    lives = {'eager': LiveRestorer(model, w=args.w, cuda_graph=False),
             'graphed': LiveRestorer(model, w=args.w, cuda_graph=True)}
    warm = frames[:6 + args.frames % 3]                           # the same last window (ring slots) as the video
    outs = {}
    for k, live in lives.items():                                 # allocation, captures of every step kind
        outs[k] = live_round(live, warm)[2]
    assert all(np.array_equal(a, b) for a, b in zip(outs['eager'], outs['graphed'])), 'graphed != eager'
    secs = {k: [] for k in lives}
    lats = {k: [] for k in lives}
    for _ in range(args.rounds):
        for k, live in lives.items():
            s, lat, _ = live_round(live, frames)
            secs[k].append(s)
            lats[k] += lat
    # one graphed steady step launches nothing through the C ABI
    g = lives['graphed']
    for f in frames[:4]:
        g.push(f)
    n = ops.launch_count()
    g.push(frames[4])
    graphed_launches = ops.launch_count() - n
    g.flush()
    live = {k: {'fps_median_round': round(args.frames / statistics.median(secs[k]), 2),
                'fps_rounds': [round(args.frames / s, 2) for s in secs[k]],
                'latency_ms': {'p50': round(1e3 * pct(lats[k], 50), 2), 'p90': round(1e3 * pct(lats[k], 90), 2),
                               'p99': round(1e3 * pct(lats[k], 99), 2), 'samples': len(lats[k])}}
            for k in lives}
    batched = {}
    for cpb in (1, 16):
        vr = VideoRestorer(model, w=args.w, clips_per_batch=cpb)
        vr.restore(frames[:2 * cpb + 1])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        vr.restore(frames)
        batched['clips_per_batch_%d' % cpb] = {'fps': round(args.frames / (time.perf_counter() - t0), 2)}
    res = {'size': args.size, 'frames': args.frames, 'rounds': args.rounds, 'w': args.w,
           'weights': args.weights or 'synthetic', 'card': card(), 'live': live, 'video_restorer': batched,
           'graphed_step_launches': graphed_launches, 'step_work': step_work(model, args.size)}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
