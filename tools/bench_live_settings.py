"""Live streams with different fidelity settings on one model (pgtformer_b200/video.py::LivePool with per-stream w and
AdaIN): one pool of S streams whose settings are mixed, the same streams split into one pool per setting (what a
service had to do before settings were per stream), and one pool whose streams share a setting, on a seeded synthetic
video, all replayed from CUDA graphs.

* settings: stream s takes SETTINGS[s % 4], (w, adain) = (1.0, on), (0.5, on), (0.3, off), (0.0, on); the uniform
  pool gives every stream (1.0, on);
* frames/s: `rounds` rounds, each streaming `frames` frames into every one of the S streams for each layout in turn (the
  three alternate within the run); aggregate = S * frames / wall time of the round (flushes included); the median
  round is reported;
* latency: host clock from the start of a step (every stream's new frame is available) to the return of the push that
  hands back that stream's restored frame, p50 / p90 over every stream and step of every round: with one pool per
  setting the pools push one after another, so a later pool's streams wait for the earlier pools' steps;
* outputs: every stream of the mixed pool equals the same stream in its own setting's pool, byte for byte;
* the card's name, power limit and max SM clock, read in the same run.

Stream s plays the video shifted by s frames.  Prints one JSON line.

    python tools/bench_live_settings.py [--streams 4,16] [--frames 30] [--size 512] [--rounds 3] [--out FILE]
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

from bench_live import build_model, pct  # noqa: E402
from bench_tdrqvae import card  # noqa: E402

SETTINGS = [(1.0, True), (0.5, True), (0.3, False), (0.0, True)]


def layout_round(pools, video, frames):
    """pools: [(pool, [(stream s, (w, adain))])]; streams frames[i + s] into stream s, every stream pushing every step,
    the pools one after another, then flushes them.  -> (seconds, [latency of every restored frame], {s: outputs})."""
    lat, outs = [], {}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    hs = [[(s, p.open(*conf)) for s, conf in streams] for p, streams in pools]
    for i in range(frames):
        a = time.perf_counter()
        for (p, _), ph in zip(pools, hs):
            r = p.push({h: video[(i + s) % len(video)] for s, h in ph})
            now = time.perf_counter()
            for s, h in ph:
                if r[h] is not None:
                    outs.setdefault(s, []).append(r[h])
                    lat.append(now - a)
    for (p, _), ph in zip(pools, hs):
        for s, h in ph:
            outs.setdefault(s, []).append(p.flush(h))
    return time.perf_counter() - t0, lat, outs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--streams', default='4,16')
    ap.add_argument('--frames', type=int, default=30, help='frames per stream and round')
    ap.add_argument('--size', type=int, default=512)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None, help='also write the JSON line to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_live_settings.py measures on a CUDA device; none found')
    from pgtformer_b200.video import LivePool
    model = build_model(None)
    video = np.random.RandomState(0).randint(0, 256, size=(args.frames + 16, args.size, args.size, 3), dtype=np.uint8)
    results = {}
    for S in [int(s) for s in args.streams.split(',')]:
        mixed = [(s, SETTINGS[s % len(SETTINGS)]) for s in range(S)]
        layouts = {
            'mixed_pool': [(LivePool(model, S), mixed)],
            'pool_per_setting': [(LivePool(model, len(own)), own) for own in
                                 ([(s, c) for s, c in mixed if c == conf] for conf in SETTINGS) if own],
            'uniform_pool': [(LivePool(model, S), [(s, SETTINGS[0]) for s in range(S)])],
        }
        warm = {k: layout_round(v, video, 5)[2] for k, v in layouts.items()}       # allocation, captures
        assert all(np.array_equal(a, b) for s in range(S)
                   for a, b in zip(warm['mixed_pool'][s], warm['pool_per_setting'][s])), 'mixed pool != own pools'
        secs = {k: [] for k in layouts}
        lats = {k: [] for k in layouts}
        for _ in range(args.rounds):
            for k, v in layouts.items():
                t, lat, _ = layout_round(v, video, args.frames)
                secs[k].append(t)
                lats[k] += lat
        res = {}
        for k, v in layouts.items():
            res[k] = {'pools': len(v), 'fps_aggregate': round(S * args.frames / statistics.median(secs[k]), 2),
                      'fps_aggregate_rounds': [round(S * args.frames / t, 2) for t in secs[k]],
                      'latency_ms': {'p50': round(1e3 * pct(lats[k], 50), 2), 'p90': round(1e3 * pct(lats[k], 90), 2),
                                     'samples': len(lats[k])},
                      'graphs': sum(len(p._state.graphs) for p, _ in v)}
        results[str(S)] = res
        del layouts, warm
        torch.cuda.empty_cache()
    line = json.dumps({'size': args.size, 'frames_per_stream': args.frames, 'rounds': args.rounds,
                       'settings': SETTINGS, 'weights': 'synthetic', 'card': card(), 'streams': results})
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
