"""PSNR / SSIM of restored frames on the device (pgt_frame_scores, pgtformer_b200/metrics.py) against the host, and
what scoring adds to restoring a video (VideoRestorer.evaluate against VideoRestorer.restore).

* `kernel`: pgt_frame_scores on 16 frame pairs of 512 x 512 and of 128 x 128, timed with CUDA events over many
  launches in alternating rounds (median).  fp64 FLOPs and bytes are counted from the shapes by `flops` / `min_bytes`
  below; the lower bound on time is the larger of FLOPs over the data sheet's fp64 rate (H100 SXM, no tensor cores)
  and bytes over its HBM3 bandwidth, and the report names which one it is.
* `host`: the same frames scored on the host by the numpy restatement of basicsr (oracle/metrics_oracle.py; basicsr's
  cv2.filter2D form where cv2 imports), one pass, wall clock.  The device scores are checked against it in the run.
* `video`: VideoRestorer(clips_per_batch=16) frames/s of restore and evaluate, for 512 x 512 frames and for 128 x 128
  sources restored at size=(512, 512), on a seeded synthetic video and synthetic weights.  Each (video, eager or
  graphed) pair is one phase whose graphs are dropped at its end, so that no more than one layout's CUDA graph pools
  are held at a time; within a phase each round runs restore and then evaluate, alternating, and the median round is
  reported.  The run checks that evaluate returns restore's bytes and that its graphed scores equal its eager ones.

The card's name, power limit and max SM clock are read in the same run.  Prints one JSON line.

    python tools/bench_metrics.py [--frames 32] [--rounds 5] [--out FILE]
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

from bench_live import build_model  # noqa: E402
from bench_tdrqvae import card  # noqa: E402

CLIPS = 16
FP64_TFLOPS, HBM_TBS = 34.0, 3.35               # H100 SXM data sheet: FP64 (non-tensor), HBM3
R = 5                                           # SSIM window radius: 11 taps


def flops(F, H, W):
    """fp64 operations of the scores as the oracle's direct separable form defines them, per channel: the products
    x^2, y^2, xy (3 H W); a horizontal then a vertical 11-tap pass of 5 fields, a multiply and an add per tap, at
    H (W - 10) and (H - 10)(W - 10) points; the map (18 operations: 3 products, 3 differences, 5 for the numerator,
    5 for the denominator, the division and the sum) at (H - 10)(W - 10) points.  The exact integer sse is not
    counted."""
    hv, vv = H * (W - 2 * R), (H - 2 * R) * (W - 2 * R)
    return 3.0 * F * (3 * H * W + 5 * (2 * R + 1) * 2 * (hv + vv) + 18 * vv)


def min_bytes(F, H, W):
    """Bytes the scores must read: both frames once."""
    return 2.0 * F * H * W * 3


def kernel_times(pairs, rounds=5, iters=50):
    from pgtformer_b200 import ops
    dev = {k: (torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()) for k, (a, b) in pairs.items()}
    ms = {k: [] for k in dev}
    for a, b in dev.values():
        ops.frame_scores(a, b)
    for _ in range(rounds):
        for k, (a, b) in dev.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                ops.frame_scores(a, b)
            e1.record()
            e1.synchronize()
            ms[k].append(e0.elapsed_time(e1) / iters)
    out = {}
    for k, (a, b) in dev.items():
        F, H, W, _ = a.shape
        t = statistics.median(ms[k]) / 1e3
        fl, by = flops(F, H, W), min_bytes(F, H, W)
        t_fl, t_by = fl / (FP64_TFLOPS * 1e12), by / (HBM_TBS * 1e12)
        out[k] = {'ms': round(t * 1e3, 4), 'ms_rounds': [round(v, 4) for v in ms[k]], 'gflop': round(fl / 1e9, 3),
                  'fp64_tflops': round(fl / t / 1e12, 2), 'mbytes': round(by / 1e6, 2),
                  'gb_s': round(by / t / 1e9, 1), 'bound': 'fp64' if t_fl >= t_by else 'hbm',
                  'share_of_bound': round(max(t_fl, t_by) / t, 3)}
    return out


def host_scores(pairs):
    """The oracle on the host, one pass per size, and the device scores checked against it."""
    from oracle import metrics_oracle as MO
    from pgtformer_b200 import metrics
    try:
        import cv2  # noqa: F401
        cv2_form = True
    except ImportError:
        cv2_form = False
    out = {}
    for k, (a, b) in pairs.items():
        t0 = time.perf_counter()
        ref = MO.score(a, b, cv2_form=cv2_form)
        secs = time.perf_counter() - t0
        got = metrics.score(a, b)
        out[k] = {'form': 'cv2.filter2D' if cv2_form else 'direct', 'seconds': round(secs, 3),
                  'ms_per_frame': round(1e3 * secs / len(a), 1),
                  'psnr_bit_identical': bool(np.array_equal(got['psnr'], ref['psnr'])),
                  'ssim_max_abs_diff': float(np.abs(got['ssim'] - ref['ssim']).max())}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=32,
                    help='frames per round of each video layout; 32 gives two batches of one shape, so one CUDA graph '
                         'per method (a 16-clip 512^2 graph holds about 17 GB)')
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--out', default=None, help='also write the JSON line to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_metrics.py measures on a CUDA device; none found')
    from pgtformer_b200 import ops
    from pgtformer_b200.video import VideoRestorer

    rs = np.random.RandomState(0)
    pairs = {}
    for s in (512, 128):
        a = rs.randint(0, 256, size=(CLIPS, s, s, 3), dtype=np.uint8)
        b = np.clip(a.astype(np.int16) + rs.randint(-12, 13, size=a.shape), 0, 255).astype(np.uint8)
        pairs['%dx%d' % (s, s)] = (a, b)
    kernel = kernel_times(pairs)
    host = host_scores(pairs)
    for k in kernel:
        kernel[k]['host_speedup'] = round(1e3 * host[k]['seconds'] / kernel[k]['ms'], 1)

    model = build_model(None)
    videos = {'512x512': (rs.randint(0, 256, size=(args.frames, 512, 512, 3), dtype=np.uint8), None),
              '128x128_to_512x512': (rs.randint(0, 256, size=(args.frames, 128, 128, 3), dtype=np.uint8), (512, 512))}
    gt = rs.randint(0, 256, size=(args.frames, 512, 512, 3), dtype=np.uint8)

    def run(vr, method, video):
        frames, size = videos[video]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = vr.restore(frames, size) if method == 'restore' else vr.evaluate(frames, gt, size)
        return time.perf_counter() - t0, res

    fps, first, launches = {}, {}, {}
    for mode, graph in (('eager', False), ('graphed', True)):
        for v in videos:                                         # one layout's graphs at a time
            vr = VideoRestorer(model, clips_per_batch=CLIPS, cuda_graph=graph)
            keys = [(v, m, mode) for m in ('restore', 'evaluate')]
            for k in keys:                                       # allocation, captures
                ops.reset_launch_count()
                first[k] = run(vr, k[1], k[0])[1]
                torch.cuda.synchronize()
                launches[k] = ops.launch_count()
                fps[k] = []
            for _ in range(args.rounds):
                for k in keys:
                    fps[k].append(args.frames / run(vr, k[1], k[0])[0])
            del vr
            model.engine().__dict__.pop('_graphs', None)
            torch.cuda.empty_cache()

    video = {}
    for v in videos:
        r = video[v] = {}
        for mode in ('eager', 'graphed'):
            med = {m: statistics.median(fps[v, m, mode]) for m in ('restore', 'evaluate')}
            r[mode] = {m: {'fps': round(med[m], 2), 'fps_rounds': [round(x, 2) for x in fps[v, m, mode]],
                           'launches_first_call': launches[v, m, mode]} for m in med}
            r[mode]['evaluate_over_restore'] = round(med['evaluate'] / med['restore'], 4)
        r['evaluate_restored_equals_restore'] = all(
            np.array_equal(first[v, 'restore', mode], first[v, 'evaluate', mode][0]) for mode in ('eager', 'graphed'))
        se, sg = first[v, 'evaluate', 'eager'][1], first[v, 'evaluate', 'graphed'][1]
        r['graphed_scores_equal_eager'] = all(np.array_equal(se[k], sg[k]) for k in ('psnr', 'ssim'))
    line = json.dumps({'card': card(), 'weights': 'synthetic', 'frames': args.frames, 'rounds': args.rounds,
                       'clips_per_batch': CLIPS, 'kernel': kernel, 'host': host, 'video': video})
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
