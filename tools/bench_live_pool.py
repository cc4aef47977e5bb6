"""Several live streams on one model (pgtformer_b200/video.py::LivePool) on a seeded synthetic video: aggregate and
per-stream frames/s and push -> output latency at S streams that all push every step, eager and replayed from CUDA
graphs, beside the batched VideoRestorer at clips_per_batch = S.

* frames/s: `rounds` rounds, each streaming `frames` frames into every one of the S streams eagerly and then graphed
  (the two alternate within the run); aggregate = S * frames / wall time of the round (flushes included), per stream =
  aggregate / S; the median round is reported;
* latency: host clock around every push that returns frames (all S restored frames in host memory when it returns),
  p50 / p90 / p99 over every such push of every round;
* C-ABI launches of one eager steady step (ops.launch_count) and of one graphed steady step (none expected), and the
  bytes the step's pgt_scatter_frames launches move, read from the C ABI's per-launch profile counters;
* VideoRestorer.restore(clips_per_batch=S) on the same frames of one stream, S * frames frames, in the same run;
* the card's name, power limit and max SM clock, read in the same run.

Stream s plays the video shifted by s frames, so the streams' frames differ.  Prints one JSON line.

    python tools/bench_live_pool.py [--streams 1,2,4,8,16] [--frames 30] [--size 512] [--rounds 3] [--w 1.0] [--out FILE]
"""
import argparse
import csv
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from bench_live import build_model, pct  # noqa: E402
from bench_tdrqvae import card  # noqa: E402


def pool_round(pool, video, S, frames):
    """Streams frames[i + s] into stream s of pool, all S streams pushing every step, then flushes them;
    -> (seconds, [latency of every push that returned frames], {stream: outputs})."""
    lat = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    hs = [pool.open() for _ in range(S)]
    outs = {h: [] for h in hs}
    for i in range(frames):
        a = time.perf_counter()
        r = pool.push({h: video[(i + s) % len(video)] for s, h in enumerate(hs)})
        if i > 0:
            lat.append(time.perf_counter() - a)
        for h, f in r.items():
            if f is not None:
                outs[h].append(f)
    for h in hs:
        outs[h].append(pool.flush(h))
    return time.perf_counter() - t0, lat, outs


def steady_step(pool, video, S):
    """Launches of one steady step (all S streams push), and the bytes of its scatter launches (profile counters)."""
    from pgtformer_b200 import ops
    hs = [pool.open() for _ in range(S)]
    for i in range(3):
        pool.push({h: video[(i + s) % len(video)] for s, h in enumerate(hs)})
    frame = {h: video[(3 + s) % len(video)] for s, h in enumerate(hs)}
    torch.cuda.synchronize()
    n = ops.launch_count()
    pool.push(frame)
    launches = ops.launch_count() - n
    scatter = None
    if not pool.cuda_graph:
        path = os.path.join(tempfile.mkdtemp(), 'step.csv')
        ops.profile_begin()
        pool.push(frame)
        ops.profile_end(path)
        with open(path) as f:
            rows = [r for r in csv.DictReader(f) if r['desc'] == 'pgt_scatter_frames']
        scatter = {'launches': len(rows), 'mbytes': round(sum(float(r['work']) for r in rows) / 1e6, 2)}
    for h in hs:
        pool.flush(h)
    return launches, scatter


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--streams', default='1,2,4,8,16')
    ap.add_argument('--frames', type=int, default=30, help='frames per stream and round')
    ap.add_argument('--size', type=int, default=512)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--w', type=float, default=1.0)
    ap.add_argument('--out', default=None, help='also write the JSON line to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_live_pool.py measures on a CUDA device; none found')
    from pgtformer_b200.video import LivePool, VideoRestorer
    model = build_model(None)
    video = np.random.RandomState(0).randint(0, 256, size=(args.frames + 16, args.size, args.size, 3), dtype=np.uint8)
    results = {}
    for S in [int(s) for s in args.streams.split(',')]:
        pools = {'eager': LivePool(model, S, w=args.w, cuda_graph=False),
                 'graphed': LivePool(model, S, w=args.w, cuda_graph=True)}
        outs = {k: pool_round(p, video, S, 5)[2] for k, p in pools.items()}     # allocation, captures
        assert all(np.array_equal(a, b) for ha, hb in zip(outs['eager'], outs['graphed'])
                   for a, b in zip(outs['eager'][ha], outs['graphed'][hb])), 'graphed != eager'
        secs = {k: [] for k in pools}
        lats = {k: [] for k in pools}
        for _ in range(args.rounds):
            for k, p in pools.items():
                s, lat, _ = pool_round(p, video, S, args.frames)
                secs[k].append(s)
                lats[k] += lat
        res = {}
        for k, p in pools.items():
            fps = S * args.frames / statistics.median(secs[k])
            launches, scatter = steady_step(p, video, S)
            res[k] = {'fps_aggregate': round(fps, 2), 'fps_per_stream': round(fps / S, 2),
                      'fps_aggregate_rounds': [round(S * args.frames / s, 2) for s in secs[k]],
                      'latency_ms': {'p50': round(1e3 * pct(lats[k], 50), 2), 'p90': round(1e3 * pct(lats[k], 90), 2),
                                     'p99': round(1e3 * pct(lats[k], 99), 2), 'samples': len(lats[k])},
                      'step_launches': launches}
            if scatter is not None:
                res[k]['step_scatter'] = scatter
        res['graphs'] = len(pools['graphed']._state.graphs)
        del pools, outs
        torch.cuda.empty_cache()
        vr = VideoRestorer(model, w=args.w, clips_per_batch=S)
        seq = video[np.arange(S * args.frames) % len(video)]
        vr.restore(seq[:2 * S + 1])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        vr.restore(seq)
        res['video_restorer_fps'] = round(len(seq) / (time.perf_counter() - t0), 2)
        results[str(S)] = res
        torch.cuda.empty_cache()
    line = json.dumps({'size': args.size, 'frames_per_stream': args.frames, 'rounds': args.rounds, 'w': args.w,
                       'weights': 'synthetic', 'card': card(), 'streams': results})
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
