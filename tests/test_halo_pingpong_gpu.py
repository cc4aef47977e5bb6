"""The ping-pong schedule of the Cout <= 128 halo convs (conv_halo_kernel<64/128, false>): each consumer warpgroup owns
alternate tiles and runs their epilogue alone.  Every case must reproduce, bit for bit, the outputs and fused GroupNorm
statistics the library recorded before that schedule (tests/golden/halo_pingpong_outputs.pt, tools/mint_halo_golden.py):
Cout 32 / 48 / 64 / 96 / 128, Cin 8 / 64 / 128 / 288 (weights resident and streamed), H and W that are not multiples of
the 16 x 8 tile, tile counts below and just above the SM count and CTAs with an odd number of tiles, bf16 / fp32 /
mixed residuals, SFT, activations, fp32 NCHW output, output into a channel slice, and the four up2x phases sharing one
statistics buffer.  The halo kernel is reached only through the ctypes binding (torch.ops.pgt has no conv op)."""
import csv
import os
import sys

import pytest
import torch

from conftest import ROOT, golden_sample, load_golden

sys.path.insert(0, os.path.join(ROOT, 'tools'))
import mint_halo_golden as M  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = load_golden('halo_pingpong_outputs.pt') if os.path.exists(
    os.path.join(ROOT, 'tests', 'golden', 'halo_pingpong_outputs.pt')) else None


def launch_descs(fn, tmp_path):
    from pgtformer_b200 import ops
    path = os.path.join(str(tmp_path), 'launches.csv')
    ops.profile_begin()
    fn()
    ops.profile_end(path)
    return [r['desc'] for r in csv.DictReader(open(path)) if r['class'] == '0']


def test_golden_covers_every_case():
    assert GOLDEN is not None
    assert [g['case']['name'] for g in GOLDEN['cases']] == [c['name'] for c in M.CASES]


@pytest.mark.parametrize('idx', range(len(M.CASES)), ids=[c['name'] for c in M.CASES])
def test_halo_bit_identical(idx, tmp_path):
    c, g = M.CASES[idx], GOLDEN['cases'][idx]
    assert g['case'] == c
    got = {}
    descs = launch_descs(lambda: got.update(M.run_case(c)), tmp_path)
    bn = 'BN64' if c['Cout'] <= 64 else 'BN128'
    assert descs and all(d.startswith('halo3 ') and (' %s ' % bn) in d for d in descs), descs
    assert len(descs) == (4 if c['kind'] == 'up2x' else 1)
    assert set(got) == {k for k in ('out', 'stats') if k in g}
    for key, t in got.items():
        s = golden_sample(t, g, key)
        assert torch.isfinite(s).all(), (c['name'], key)
        assert torch.equal(s, g[key]), '%s/%s: %d of %d sampled elements differ' % (
            c['name'], key, int((s != g[key]).sum()), s.numel())
