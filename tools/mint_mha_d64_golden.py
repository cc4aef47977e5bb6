"""Records the d = 64 outputs of `pgt_mha_fwd` (mha_tc.cu, and the mma.sync kernel for L not a multiple of 128) on
seeded inputs, for tests/test_attn_wide_gpu.py::test_d64_unchanged: run with the library as it was before the wide-head
kernel was added, so the test shows that path unchanged bit for bit.

tests/golden/mha_d64_outputs.pt was recorded on an H100 with the library built at commit
7110ee72dc8fecce23fb23afc7a2c9292ff2bde2 (the commit before attn_wide_tc.cu); the file stores that id as
`library_commit`.  To reproduce it, check out that commit, build it, and run this script from the newer tree with the
old package first on the path:

    PYTHONPATH=<old checkout> python tools/mint_mha_d64_golden.py OUT.pt --commit <id of the old checkout>
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.append(ROOT)

CASES = ((2, 128, 8, 500), (1, 200, 8, 510), (1, 384, 4, 520))      # (clips, L, heads, seed)


def rnd(shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g).to(torch.bfloat16).to('cuda')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('out')
    ap.add_argument('--commit', required=True, help='commit the loaded library was built from')
    args = ap.parse_args()
    from pgtformer_b200 import ops
    cases = []
    for clips, L, heads, seed in CASES:
        q, k, v = (rnd((clips * L, heads * 64), seed + i) for i in range(3))
        out = torch.empty(clips * L, heads * 64, dtype=torch.bfloat16, device='cuda')
        ops.mha(q, k, v, clips, L, heads, 64, out)
        torch.cuda.synchronize()
        cases.append({'clips': clips, 'L': L, 'heads': heads, 'seed': seed, 'out': out.cpu()})
    torch.save({'cases': cases, 'library_commit': args.commit}, args.out)


if __name__ == '__main__':
    main()
