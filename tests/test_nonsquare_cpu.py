"""CPU tests: the oracle restatement against the reference at frames with H != W (oracle/make_golden.py --nonsquare).
With one 64-pixel side, level 4 and the mid layers are one window row (or column) deep: the reference's
get_window_size then drops the shift of that axis only, and the shifted blocks still roll and mask the other."""
import pytest
import torch

from conftest import golden_sample, load_golden
from oracle import pgt_oracle as O
from oracle.make_golden import NONSQUARE_CASES, golden_input, nonsquare_name

TOL = 2e-5      # as tests/test_oracle.py: fp32 summation-order noise between two CPU formulations
FIXTURES = [nonsquare_name(*c) for c in NONSQUARE_CASES]


@pytest.mark.parametrize('fixture', FIXTURES)
def test_oracle_matches_reference_golden_nonsquare(arch_spec, synth_sd, fixture):
    arch, _ = arch_spec
    g = load_golden(fixture)
    assert g['H'] != g['W']
    x = golden_input(g['seed'], g['b'], g['H'], g['W'])
    with torch.no_grad():
        out, logits, lq = O.pgtformer_forward(synth_sd, arch, x, w=g['w'], adain_on=g['adain'])
        vq_out, _, vq_codes = O.tdcrqvae3_forward(synth_sd, arch, x)
    assert (golden_sample(lq, g, 'lq_feat') - g['lq_feat']).abs().max() < TOL
    assert (golden_sample(logits, g, 'logits') - g['logits']).abs().max() < TOL
    assert (golden_sample(out, g, 'out') - g['out']).abs().max() < TOL * 10
    assert torch.equal(logits.argmax(-1), g['codes'])
    assert torch.equal(vq_codes, g['vq_codes'])
    assert (golden_sample(vq_out, g, 'vq_out') - g['vq_out']).abs().max() < TOL * 10


@pytest.mark.parametrize('H,W,shifts', [(4, 12, (0, 2)), (12, 4, (2, 0)), (4, 4, (0, 0)), (8, 8, (2, 2)),
                                        (8, 4, (2, 0))])
def test_window_shift_is_per_axis(H, W, shifts):
    """get_window_size (`modules/rstt_layers.py:90-114`) decides each axis alone; the mask separates only the regions
    of the shifted axes: 2 window patterns per shifted axis (interior, wrapped)."""
    assert O.window_shift(H, W) == shifts
    m = O.shift_mask(H, W)
    assert m.shape == ((H // 4) * (W // 4), 48, 48)
    patterns = {tuple(w.flatten().tolist()) for w in m}
    assert len(patterns) == (2 if shifts[0] else 1) * (2 if shifts[1] else 1)
    if shifts != (0, 0):
        assert set(m.unique().tolist()) == {0.0, -100.0}


def test_oracle_codec_matches_reference_golden_nonsquare(arch_spec, synth_sd):
    from oracle import codec_oracle as C
    arch, _ = arch_spec
    g = load_golden('tdcrqvae3_codec_b1_64x192_seed23.pt')
    x = golden_input(g['seed'], g['b'], g['H'], g['W'])
    cb = synth_sd['quantizer.codebooks.0.weight']
    with torch.no_grad():
        z_e = C.tdcrqvae3_encode(synth_sd, arch, x)
        out = C.tdcrqvae3_decode(synth_sd, arch, O.embed_code(cb, g['codes']))
        out_code = C.tdcrqvae3_decode(synth_sd, arch, O.embed_code(cb, g['code']))
    assert (golden_sample(z_e, g, 'z_e') - g['z_e']).abs().max() < TOL
    assert torch.equal(O.l2_argmin(cb, z_e).unsqueeze(-1), g['codes'])
    assert (golden_sample(out, g, 'out') - g['out']).abs().max() < TOL * 10
    assert int(g['code'].max()) == cb.shape[0] - 1                 # the padding row is part of the code map
    assert (golden_sample(out_code, g, 'out_code') - g['out_code']).abs().max() < TOL * 10
