"""The `lr` protocol of the reference's test set from ground truth alone (pgtformer_b200/degrade.py,
VideoRestorer.evaluate(gt, gt, downscale=0.25)) on a seeded synthetic 512 x 512 video and synthetic weights.

* `kernel`: CUDA-event times of the device degradation, pgt_imresize_u8hwc_to_f32nchw (16 frames 512^2 -> 128^2)
  plus pgt_f32nchw_resize_to_f32nchw (128^2 -> 512^2), against pgt_u8hwc_resize_to_f32nchw (16 frames of 128^2 ->
  512^2, the `LR_Blind` input), in alternating rounds; median ms per launch.
* `evaluate_eager` / `evaluate_graphed`: VideoRestorer(clips_per_batch=16).evaluate(gt, gt, downscale=0.25) frames/s.
* `host`: the route without this module: basicsr's imresize in torch float32 on the CPU (oracle/degrade_oracle.py's
  reference form), F.interpolate on the CPU, the fp32 windows copied to the device from pinned memory and restored by
  one batched PGTFormer.forward per 16 windows, then scored with metrics.score.  Its model inputs and restored bytes
  are compared with the device route's: basicsr's `mv` rounds each sum in its BLAS's order, the device once from the
  exact sum, so the inputs differ in the last bits; the outputs then differ wherever that moves a code's argmax (the
  quantiser is discontinuous, and synthetic weights put many logits close together).

Every round runs every layout once, alternating; the median round is reported.  The card's name, power limit and
max SM clock are read in the same run.  Prints one JSON line.

    python tools/bench_lr_degrade.py [--frames 32] [--rounds 3] [--out FILE]
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

from bench_live import build_model  # noqa: E402
from bench_tdrqvae import card  # noqa: E402

GT, LR, CLIPS, SCALE = (512, 512), (128, 128), 16, 0.25


def host_route(model, gt):
    """The host route: basicsr-form imresize and F.interpolate on the CPU, batched forward, metrics.score."""
    from oracle import degrade_oracle as DO
    from pgtformer_b200 import metrics, ops
    from pgtformer_b200.video import window_indices
    eng = model.engine()
    lq = torch.from_numpy(DO.lr_basicsr(gt, SCALE))
    lq = F.interpolate(lq, GT, mode='bilinear', align_corners=True)
    wins = window_indices(len(gt))
    out = np.empty(gt.shape, np.uint8)
    for first in range(0, len(gt), CLIPS):
        idx = [j for win in wins[first:first + CLIPS] for j in win]
        x = lq[idx].pin_memory().to(eng.dev, non_blocking=True)
        y = eng.forward(x)[0]
        n = len(idx) // 3
        res = ops.f32nchw_to_u8hwc(y, torch.empty((n,) + GT + (3,), dtype=torch.uint8, device=eng.dev), 1, 3)
        out[first:first + n] = res.cpu().numpy()
    return out, metrics.score(out, gt)


def input_diff(gt):
    """The model inputs of both routes: max |host - device| and the share of values that differ."""
    from oracle import degrade_oracle as DO
    from pgtformer_b200 import degrade, ops
    host = F.interpolate(torch.from_numpy(DO.lr_basicsr(gt, SCALE)), GT, mode='bilinear', align_corners=True)
    lo = degrade.downsample(gt, SCALE)
    dev = ops.f32nchw_resize_to_f32nchw(lo, torch.empty((len(gt), 3) + GT, device='cuda')).cpu()
    d = (host.double() - dev.double()).abs()
    return {'input_max_abs_diff': float(d.max()), 'input_values_differing': round(float((d > 0).double().mean()), 4)}


def kernel_times(rounds=5, iters=50):
    from pgtformer_b200 import degrade, ops
    gt = torch.randint(0, 256, (CLIPS,) + GT + (3,), dtype=torch.uint8, device='cuda')
    lo = torch.randint(0, 256, (CLIPS,) + LR + (3,), dtype=torch.uint8, device='cuda')
    small = torch.empty((CLIPS, 3) + LR, device='cuda')
    out = torch.empty((CLIPS, 3) + GT, device='cuda')

    def lr():
        degrade.resize(gt, SCALE, small)
        ops.f32nchw_resize_to_f32nchw(small, out)
    runs = {'imresize_512_to_128': lambda: degrade.resize(gt, SCALE, small),
            'imresize_plus_resize_to_512': lr,
            'u8hwc_resize_128_to_512': lambda: ops.u8hwc_resize_to_f32nchw(lo, out, LR)}
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
    return {k: round(statistics.median(v), 4) for k, v in ms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=32)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None, help='also write the JSON line to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_lr_degrade.py measures on a CUDA device; none found')
    from pgtformer_b200.video import VideoRestorer
    model = build_model(None)
    gt = np.random.RandomState(0).randint(0, 256, size=(args.frames,) + GT + (3,), dtype=np.uint8)
    gt[:, :, ::32] = 255                                  # step edges, so the low-resolution frames overshoot
    layouts = {'evaluate_eager': VideoRestorer(model, clips_per_batch=CLIPS).evaluate,
               'evaluate_graphed': VideoRestorer(model, clips_per_batch=CLIPS, cuda_graph=True).evaluate,
               'host': None}

    def run(name):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        got = host_route(model, gt) if name == 'host' else layouts[name](gt, gt, downscale=SCALE)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, got

    first = {k: run(k)[1] for k in layouts}
    fps = {k: [] for k in layouts}
    for _ in range(args.rounds):
        for k in layouts:
            fps[k].append(args.frames / run(k)[0])
    dev_out, dev_scores = first['evaluate_eager']
    host_out, host_scores = first['host']
    diff = np.abs(dev_out.astype(int) - host_out.astype(int))
    res = {k: {'fps': round(statistics.median(v), 2), 'fps_rounds': [round(x, 2) for x in v]} for k, v in fps.items()}
    line = json.dumps({
        'ground_truth': list(GT), 'scale': SCALE, 'frames': args.frames, 'rounds': args.rounds, 'weights': 'synthetic',
        'card': card(), 'layouts': res, 'kernel_ms': kernel_times(),
        'graphed_equals_eager': bool(np.array_equal(dev_out, first['evaluate_graphed'][0])),
        'host_vs_device': {'max_abs_diff': int(diff.max()), 'bytes_differing': int((diff > 0).sum()),
                           'bytes': int(diff.size),
                           'max_psnr_diff_db': float(np.abs(dev_scores['psnr'] - host_scores['psnr']).max()),
                           'max_ssim_diff': float(np.abs(dev_scores['ssim'] - host_scores['ssim']).max()),
                           **input_diff(gt)},
        'h2d_bytes_per_frame': {'evaluate': 2 * GT[0] * GT[1] * 3, 'host': 3 * 3 * GT[0] * GT[1] * 4}})
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
