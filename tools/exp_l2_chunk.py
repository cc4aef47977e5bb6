#!/usr/bin/env python
"""Experiment: depth-first (frame-chunked) execution of an attention-free level.  GroupNorm statistics are per frame, so
a chain conv -> GN apply -> conv -> ... can run on a few frames at a time; with a chunk whose tensors fit the 50 MB L2
the intermediate tensors are re-read from L2 instead of HBM.  Times the decoder's 512^2 and 256^2 res-block chains for
several chunk sizes (CUDA events, whole chain, 48 frames).
    python tools/exp_l2_chunk.py
"""
import os
import sys

import torch
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from archs.pgtformer_arch import PGTFormer  # noqa: E402

DEV = 'cuda:0'


def frames(t, f0, f1):
    s = t[f0:f1]
    gn = getattr(t, '_pgt_gn', None)
    if gn is not None:
        st = gn[0].view(t.shape[0], -1)[f0:f1].reshape(-1)
        s._pgt_gn = (st, gn[1])
    return s


def main():
    with open(os.path.join(ROOT, 'options', 'release_test_stage_IIII_dont_need_align_version.yml')) as f:
        opt = yaml.safe_load(f)['network_g']
    kw = dict(opt)
    kw.pop('type')
    model = PGTFormer(**kw).to(DEV)
    model.eval()
    E = model.engine()
    Fr = 48
    for (H, C, lvl) in ((512, 64, 0), (256, 128, 1)):
        x0 = (torch.randn(Fr, H, H, C, device=DEV) * 0.5).bfloat16()
        blocks = ['decoder.up.%d.block.%d' % (lvl, b) for b in (1, 1)]

        def chain(x):
            for p in blocks:
                x = E.td_resblock(x, p, C, gn_next=True)
            return x

        with torch.no_grad(), torch.cuda.device(DEV):
            x = E.td_resblock(x0, blocks[0], C, gn_next=True)      # carries GroupNorm statistics
            ref = chain(x)
            torch.cuda.synchronize()
            for chunk in (48, 6, 3, 2, 1):
                def run():
                    outs = []
                    for f0 in range(0, Fr, chunk):
                        outs.append(chain(frames(x, f0, f0 + chunk)))
                    return outs
                for _ in range(2):
                    outs = run()
                torch.cuda.synchronize()
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    outs = run()
                torch.cuda.synchronize()
                graph.replay()
                torch.cuda.synchronize()
                same = all(torch.equal(o, ref[i * chunk:(i + 1) * chunk]) for i, o in enumerate(outs))
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                iters = 3
                e0.record()
                for _ in range(iters):
                    graph.replay()
                e1.record()
                torch.cuda.synchronize()
                print('H=%d C=%d chunk=%2d frames: %.3f ms per chain of 2 res blocks (48 frames), identical=%s' %
                      (H, C, chunk, e0.elapsed_time(e1) / iters, same), flush=True)


if __name__ == '__main__':
    main()
