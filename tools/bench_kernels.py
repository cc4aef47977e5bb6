#!/usr/bin/env python
"""Micro-benchmarks of the north_star kernels through the C ABI (CUDA events, warm-up, inputs larger than L2 or an L2
flush between iterations): window attention (mma.sync round-1 kernel vs TMA + wgmma), L2 argmin (FFMA vs wgmma),
row argmax + gather.  Prints one JSON line per case: achieved GB/s and TFLOP/s against MEASURED_PEAKS.json.
    python tools/bench_kernels.py [--quick]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pgtformer_b200 import ops  # noqa: E402
from pgtformer_b200.weights import relative_position_index  # noqa: E402

DEV = 'cuda'


def peaks():
    p = os.path.join(ROOT, 'MEASURED_PEAKS.json')
    if os.path.exists(p):
        return json.load(open(p))
    return {'hbm_gbs': 6650.0, 'bf16_tflops': 1590.0, 'bf16_tflops_sustained': 1400.0}


_flush = None


def flush_l2():
    global _flush
    if _flush is None:
        _flush = torch.empty(256 << 20, dtype=torch.uint8, device=DEV)
    _flush.zero_()


def timed(fn, iters=10, warm=3, flush=True):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    tot = 0.0
    for _ in range(iters):
        if flush:
            flush_l2()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
    return tot / iters


def bench_window(C, H, clips, shift, pk, out):
    heads = 8
    T = clips * 3 * H * H
    g = torch.Generator().manual_seed(1)
    qkv = torch.randn(T, 3 * C, generator=g).bfloat16().to(DEV)
    table = 0.5 * torch.randn(245, heads, generator=g)
    bias = table[relative_position_index().view(-1)].view(48, 48, heads).permute(2, 0, 1).contiguous().to(DEV)
    tab16 = ops.window_tables(bias)
    o = torch.empty(T, C, dtype=torch.bfloat16, device=DEV)
    bytes_ = T * 4 * C * 2                                        # read q,k,v + write o (SURVEY 8d)
    flops = 4.0 * 48 * 48 * C * (T // 48)
    cases = [('mma_sync', lambda: ops.window_attention(qkv, clips, H, H, C, heads, shift, bias, o)),
             ('wgmma', lambda: ops.window_attention_tc(qkv, clips, H, H, C, heads, shift, tab16, o, mode_n64=0))]
    if C // heads == 32:
        cases.append(('wgmma_n64', lambda: ops.window_attention_tc(qkv, clips, H, H, C, heads, shift, tab16, o, mode_n64=1)))
    for name, fn in cases:
        ms = timed(fn)
        out({'kernel': 'window_attention', 'impl': name, 'C': C, 'H': H, 'clips': clips, 'shift': shift, 'ms': ms,
             'GBps': bytes_ / ms / 1e6, 'hbm_frac': bytes_ / ms / 1e6 / pk['hbm_gbs'], 'TFLOPs': flops / ms / 1e9})


def bench_argmin(T, regime, pk, out, with_ffma=True):
    g = torch.Generator().manual_seed(2)
    cb = torch.randn(1025, 512, generator=g).to(DEV)
    if regime == 'near_code':
        pick = torch.randint(0, 1024, (T,), generator=g).to(DEV)
        z = cb[pick] + 0.05 * torch.randn(T, 512, generator=g).to(DEV)
    else:
        z = torch.randn(T, 512, generator=g).to(DEV)
    z = z.contiguous()
    idx = torch.empty(T, dtype=torch.int64, device=DEV)
    quant = torch.empty(T, 512, dtype=torch.float32, device=DEV)
    pack = ops.codebook_pack(cb, 1024)
    flops = 2.0 * T * 1024 * 512
    bytes_ = T * 512 * 4 + 1024 * 512 * 4 + T * 8                 # SURVEY 8(d): z fp32 + codebook + indices
    cases = [('wgmma', lambda: ops.l2_argmin_tc(z, cb, pack, 1024, idx, None)),
             ('wgmma+quant', lambda: ops.l2_argmin_tc(z, cb, pack, 1024, idx, quant))]
    if with_ffma:
        cases.append(('fp64_exhaustive', lambda: ops.l2_argmin(z, cb, 1024, idx, None)))
    for name, fn in cases:
        ms = timed(fn, iters=5 if name == 'fp64_exhaustive' else 10)
        # device time of the sweep kernel alone (events around the launch inside the library)
        ops.profile_begin()
        for _ in range(5):
            flush_l2()
            fn()
        prof = ops.profile_end()
        kms = prof['l2_argmin'][1] / max(prof['l2_argmin'][2], 1)
        out({'kernel': 'l2_argmin', 'impl': name, 'T': T, 'regime': regime, 'ms': ms, 'kernel_ms': kms,
             'TFLOPs': flops / kms / 1e9, 'tensor_frac_burst': flops / kms / 1e9 / pk['bf16_tflops'],
             'GBps': bytes_ / kms / 1e6, 'hbm_frac': bytes_ / kms / 1e6 / pk['hbm_gbs'],
             'fallback_tokens': int(ops.last_l2_argmin_fallbacks())})


def bench_argmax(T, pk, out):
    g = torch.Generator().manual_seed(3)
    logits = torch.randn(T, 1024, generator=g).to(DEV)
    cb = torch.randn(1025, 512, generator=g).to(DEV)
    idx = torch.empty(T, dtype=torch.int64, device=DEV)
    quant = torch.empty(T, 512, dtype=torch.float32, device=DEV)
    bytes_ = T * 1024 * 4 + T * 8 + T * 512 * 4
    ms = timed(lambda: ops.argmax_gather(logits, cb, idx, quant))
    out({'kernel': 'argmax_gather', 'T': T, 'ms': ms, 'GBps': bytes_ / ms / 1e6, 'hbm_frac': bytes_ / ms / 1e6 / pk['hbm_gbs']})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--quick', action='store_true')
    ap.add_argument('--only', default='')
    a = ap.parse_args()
    pk = peaks()

    def out(d):
        print(json.dumps(d), flush=True)

    if a.only in ('', 'window'):
        for (C, H, clips) in ((256, 128, 16), (256, 64, 16), (512, 32, 16)) if not a.quick else ((256, 128, 4),):
            for shift in (0, 2):
                bench_window(C, H, clips, shift, pk, out)
    if a.only in ('', 'argmin'):
        for T in (49152, 98304) if not a.quick else (49152,):
            for regime in ('random', 'near_code'):
                bench_argmin(T, regime, pk, out, with_ffma=(T == 49152))
    if a.only in ('', 'argmax'):
        bench_argmax(49152, pk, out)


if __name__ == '__main__':
    main()
