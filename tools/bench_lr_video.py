"""Low-resolution face video restored at the model's size (pgtformer_b200/video.py, size=...) on a seeded synthetic
video and synthetic weights: 128 x 128 rgb24 sources restored at 512 x 512, each frame upsampled on the device as the
reference's test set feeds its LR_Blind frames to the model (data/vfhq_full_dataset.py:1046-1051).

Layouts, each eager and replayed from CUDA graphs:
* `video_restorer`: VideoRestorer(clips_per_batch=16).restore(frames, size=(512, 512)) over `frames` frames;
* `pool_S`: LivePool(S, size=(512, 512)), S streams all pushing every step, `frames` frames each (flushes included);
* `fp32_host`: the route without `size`: each batch of 16 windows upsampled on the host with F.interpolate to fp32,
  copied to the device from pinned memory and restored by one batched PGTFormer.forward (graphed: forward_graphed),
  the middle frames converted back to rgb24 on the device.

Eager layouts are measured in one phase and graphed ones in a second (their CUDA graphs' memory pools do not fit
beside the eager caches at 16 streams and 16 clips); within a phase every round runs every layout once, alternating,
and the median round is reported: frames/s, and for the pools the
p50 / p90 push -> output latency over every push of every round.  H2D bytes per frame are counted from the shapes of
what each layout copies.  The upsampling kernel is timed with CUDA events against pgt_u8hwc_to_f32nchw writing the
same output size (16 frames of 512 x 512), in alternating rounds.  The card's name, power limit and max SM clock are
read in the same run.  Prints one JSON line.

    python tools/bench_lr_video.py [--frames 32] [--rounds 3] [--streams 1,4,16] [--out FILE]
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from bench_live import build_model, pct  # noqa: E402
from bench_live_pool import pool_round  # noqa: E402
from bench_tdrqvae import card  # noqa: E402

SRC, SIZE, CLIPS = (128, 128), (512, 512), 16


class HostFp32:
    """The fp32 route: windows upsampled on the host, one batched forward per CLIPS windows."""

    def __init__(self, model, graphed):
        self.model, self.graphed = model, graphed

    def restore(self, frames, size):
        from pgtformer_b200 import ops
        from pgtformer_b200.video import window_indices
        eng = self.model.engine()
        wins = window_indices(len(frames))
        out = np.empty((len(frames),) + size + (3,), np.uint8)
        for first in range(0, len(frames), CLIPS):
            idx = [j for win in wins[first:first + CLIPS] for j in win]
            lq = torch.from_numpy(np.array(frames[idx] / 255.0, np.float32)).permute(0, 3, 1, 2)
            x = F.interpolate(lq, size, mode='bilinear', align_corners=True).pin_memory().to(eng.dev, non_blocking=True)
            y = (eng.forward_graphed(x) if self.graphed else eng.forward(x))[0]
            n = len(idx) // 3
            res = ops.f32nchw_to_u8hwc(y, torch.empty((n,) + size + (3,), dtype=torch.uint8, device=eng.dev), 1, 3)
            out[first:first + n] = res.cpu().numpy()
        return out


def h2d_bytes_per_frame(name, n):
    """Bytes a layout copies host -> device per restored frame, from the shapes it copies."""
    from pgtformer_b200.video import plan_batches
    src = SRC[0] * SRC[1] * 3
    if name == 'video_restorer':                       # a batch stages its distinct frames lo..hi; int32 window index
        return sum((hi - lo + 1) * src + 12 * cnt for _, cnt, lo, hi in plan_batches(n, CLIPS)) / n
    if name == 'fp32_host':                            # three fp32 frames per window
        return 3 * 3 * SIZE[0] * SIZE[1] * 4
    return src + 13 * 4                                # the source frame; 13 S int32 step inputs shared by S frames


def kernel_times(rounds=5, iters=50):
    """Median ms per launch of the upsampling (16 frames of 128^2 -> 512^2) and of pgt_u8hwc_to_f32nchw (16 frames
    of 512^2), timed with CUDA events in alternating rounds."""
    from pgtformer_b200 import ops
    lo = torch.randint(0, 256, (CLIPS,) + SRC + (3,), dtype=torch.uint8, device='cuda')
    hi = torch.randint(0, 256, (CLIPS,) + SIZE + (3,), dtype=torch.uint8, device='cuda')
    out = torch.empty((CLIPS, 3) + SIZE, device='cuda')
    runs = {'resize_128_to_512': lambda: ops.u8hwc_resize_to_f32nchw(lo, out, SRC),
            'u8hwc_to_f32nchw_512': lambda: ops.u8hwc_to_f32nchw(hi, out)}
    ms = {k: [] for k in runs}
    for f in runs.values():
        f()
    for _ in range(rounds):
        for k, f in runs.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                f()
            b.record()
            b.synchronize()
            ms[k].append(a.elapsed_time(b) / iters)
    written = CLIPS * 3 * SIZE[0] * SIZE[1] * 4
    return {k: {'ms': round(statistics.median(v), 4), 'written_gb_s': round(written / statistics.median(v) / 1e6, 1)}
            for k, v in ms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=32, help='frames per round (per stream for the pools)')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--streams', default='1,4,16')
    ap.add_argument('--out', default=None, help='also write the JSON line to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_lr_video.py measures on a CUDA device; none found')
    from pgtformer_b200.video import LivePool, VideoRestorer
    model = build_model(None)
    video = np.random.RandomState(0).randint(0, 256, size=(args.frames + 16,) + SRC + (3,), dtype=np.uint8)
    seq = video[:args.frames]
    streams = [int(s) for s in args.streams.split(',')]

    def run(key, obj):
        """-> (seconds, frames restored, push latencies, outputs)."""
        if key[0].startswith('pool_'):
            S = int(key[0][5:])
            secs, lat, outs = pool_round(obj, video, S, args.frames)
            return secs, S * args.frames, lat, [np.stack(o) for o in outs.values()]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = obj.restore(seq, SIZE)
        return time.perf_counter() - t0, len(seq), [], [out]

    fps, lats, first = {}, {}, {}
    # Eager layouts in one phase, graphed ones in a second: the graphs' memory pools do not fit beside the eager
    # caches at 16 streams and 16 clips.
    for mode, graph in (('eager', False), ('graphed', True)):
        layouts = {('video_restorer', mode): VideoRestorer(model, clips_per_batch=CLIPS, cuda_graph=graph),
                   ('fp32_host', mode): HostFp32(model, graph)}
        for S in streams:
            layouts['pool_%d' % S, mode] = LivePool(model, S, cuda_graph=graph, size=SIZE)
        for k, o in layouts.items():                               # allocation, captures
            first[k] = run(k, o)[3]
            fps[k], lats[k] = [], []
        for _ in range(args.rounds):
            for k, o in layouts.items():
                secs, n, lat, _ = run(k, o)
                fps[k].append(n / secs)
                lats[k] += lat
        del layouts
        model.engine().__dict__.pop('_graphs', None)
        torch.cuda.empty_cache()
    same = {k: all(np.array_equal(a, b) for a, b in zip(first[k, 'eager'], first[k, 'graphed']))
            for k, _ in first}
    fp32_vs_lr = int(np.abs(first['video_restorer', 'eager'][0].astype(int)
                            - first['fp32_host', 'eager'][0].astype(int)).max())
    res = {}
    for (name, mode), v in fps.items():
        r = res.setdefault(name, {'graphed_equals_eager': same[name]})
        r[mode] = {'fps': round(statistics.median(v), 2), 'fps_rounds': [round(x, 2) for x in v]}
        if name.startswith('pool_'):
            lat = lats[name, mode]
            r[mode]['latency_ms'] = {'p50': round(1e3 * pct(lat, 50), 2), 'p90': round(1e3 * pct(lat, 90), 2),
                                     'samples': len(lat)}
        r['h2d_bytes_per_frame'] = round(h2d_bytes_per_frame(name, args.frames))
    line = json.dumps({'source': list(SRC), 'size': list(SIZE), 'frames': args.frames, 'rounds': args.rounds,
                       'weights': 'synthetic', 'card': card(), 'layouts': res,
                       'fp32_host_max_abs_diff_vs_size_path': fp32_vs_lr, 'kernel': kernel_times()})
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
