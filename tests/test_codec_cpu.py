"""CPU tests of the stage-I codec methods (TDCRQVAE3.encode / decode / decode_code / get_soft_codes): the oracle's
restatements against outputs of the reference's own methods (tests/golden/tdcrqvae3_codec_*.pt, minted by
`python -m oracle.make_codec_golden`), and the argument checks the model does on the host before any launch."""
import math

import pytest
import torch

from conftest import golden_sample, load_golden
from oracle import codec_oracle as C
from oracle import pgt_oracle as O
from oracle.make_golden import golden_input

TOL = 2e-5      # as tests/test_oracle.py: fp32 summation-order noise between two CPU formulations


def test_oracle_codec_matches_reference_golden_64(arch_spec, synth_sd):
    arch, _ = arch_spec
    g = load_golden('tdcrqvae3_codec_b1_64_seed21.pt')
    x = golden_input(g['seed'], g['b'], g['H'])
    cb = synth_sd['quantizer.codebooks.0.weight']
    with torch.no_grad():
        z_e = C.tdcrqvae3_encode(synth_sd, arch, x)
        out = C.tdcrqvae3_decode(synth_sd, arch, g['z_q'])
        out_code = C.tdcrqvae3_decode(synth_sd, arch, O.embed_code(cb, g['code']))
    assert z_e.shape == g['z_e'].shape and (z_e - g['z_e']).abs().max() < TOL
    assert torch.equal(O.l2_argmin(cb, z_e).unsqueeze(-1), g['codes'])
    assert out.shape == g['out'].shape and (out - g['out']).abs().max() < TOL * 10
    assert int(g['code'].max()) == cb.shape[0] - 1                 # the padding row is part of the code map
    assert (out_code - g['out_code']).abs().max() < TOL * 10


def test_oracle_soft_codes_match_reference_golden(arch_spec, synth_sd):
    arch, _ = arch_spec
    g = load_golden('tdcrqvae3_codec_soft_b1_64_seed21.pt')
    x = golden_input(g['seed'], g['b'], g['H'])
    cb = synth_sd['quantizer.codebooks.0.weight']
    with torch.no_grad():
        z_e = C.tdcrqvae3_encode(synth_sd, arch, x)
    assert tuple(g['temps']) == (1.0, 10.0, 100.0)
    for t, ref, rcode in zip(g['temps'], g['soft_code'], g['code']):
        p, code = C.soft_codes(cb, z_e, t)
        assert p.shape == ref.shape == (3, 4, 4, 1, 1024)
        assert (p - ref).abs().max() < TOL
        assert torch.equal(code, rcode)


def test_oracle_codec_matches_reference_golden_128_b2(arch_spec, synth_sd):
    arch, _ = arch_spec
    g = load_golden('tdcrqvae3_codec_b2_128_seed22.pt')
    x = golden_input(g['seed'], g['b'], g['H'])
    cb = synth_sd['quantizer.codebooks.0.weight']
    with torch.no_grad():
        z_e = C.tdcrqvae3_encode(synth_sd, arch, x)
        out = C.tdcrqvae3_decode(synth_sd, arch, O.embed_code(cb, g['codes']))
    assert (golden_sample(z_e, g, 'z_e') - g['z_e']).abs().max() < TOL
    assert torch.equal(O.l2_argmin(cb, z_e).unsqueeze(-1), g['codes'])
    assert (golden_sample(out, g, 'out') - g['out']).abs().max() < TOL * 10


# --------------------------------------------------------------------------- host-side argument checks
@pytest.fixture(scope='module')
def cpu_model(network_g):
    from archs.pgtformer_arch import PGTFormer
    opt = dict(network_g)
    opt.pop('type')
    return PGTFormer(**opt)


@pytest.mark.parametrize('temp', [0.0, -1.0, math.nan, math.inf, -math.inf, 'warm', None])
def test_get_soft_codes_rejects_bad_temperature(cpu_model, temp):
    with pytest.raises(ValueError):
        cpu_model.get_soft_codes(torch.rand(3, 3, 64, 64), temp=temp)


@pytest.mark.parametrize('shape', [(3, 64, 64), (2, 3, 64, 64), (3, 4, 64, 64), (3, 3, 48, 64), (3, 3, 64, 80),
                                   (1, 2, 3, 64, 64), (1, 1, 3, 3, 64, 64)])
def test_frame_inputs_reject_bad_shapes(cpu_model, shape):
    x = torch.rand(*shape)
    for call in (cpu_model.encode, cpu_model.get_soft_codes, lambda v: cpu_model.forward_partial_code(v, 0)):
        with pytest.raises(ValueError):
            call(x)


@pytest.mark.parametrize('shape', [(3, 4, 4), (3, 4, 4, 256), (2, 4, 4, 512), (3, 6, 4, 512), (3, 4, 4, 512, 1)])
def test_decode_rejects_bad_shapes(cpu_model, shape):
    with pytest.raises(ValueError):
        cpu_model.decode(torch.zeros(*shape))


@pytest.mark.parametrize('code', [torch.zeros(3, 4, 4, dtype=torch.int64), torch.zeros(3, 4, 4, 2, dtype=torch.int64),
                                  torch.zeros(3, 4, 4, 1), torch.zeros(2, 4, 4, 1, dtype=torch.int64),
                                  torch.zeros(3, 4, 6, 1, dtype=torch.int64)])
def test_decode_code_rejects_bad_shapes(cpu_model, code):
    with pytest.raises(ValueError):
        cpu_model.decode_code(code)


@pytest.mark.parametrize('bad', [-1, 1025, 1 << 40])
def test_codes_out_of_range_raise_index_error(cpu_model, bad):
    code = torch.zeros(3, 4, 4, 1, dtype=torch.int64)
    code[1, 2, 3, 0] = bad
    for call in (cpu_model.decode_code, cpu_model.get_code_emb_with_depth, lambda c: cpu_model.decode_partial_code(c, 0)):
        with pytest.raises(IndexError):
            call(code)


def test_partial_code_arguments(cpu_model):
    code = torch.zeros(3, 4, 4, 1, dtype=torch.int64)
    with pytest.raises(AssertionError):
        cpu_model.decode_partial_code(code, 1)                      # code_idx >= depth, as the reference asserts
    with pytest.raises(NotImplementedError):
        cpu_model.decode_partial_code(code, 0, decode_type='mean')


def test_valid_arguments_on_a_cpu_model_raise_no_cpu_path(cpu_model):
    """Checks pass, then the engine refuses to run on the CPU (code 1024, the padding row, is valid)."""
    code = torch.full((3, 4, 4, 1), 1024, dtype=torch.int64)
    calls = (lambda: cpu_model.encode(torch.rand(3, 3, 64, 64)), lambda: cpu_model.decode(torch.zeros(3, 4, 4, 512)),
             lambda: cpu_model.decode_code(code), lambda: cpu_model.get_code_emb_with_depth(code),
             lambda: cpu_model.decode_partial_code(code, 0, 'add'),
             lambda: cpu_model.get_soft_codes(torch.rand(1, 3, 3, 64, 64), temp=0.5, stochastic=True))
    for call in calls:
        with pytest.raises(RuntimeError, match='no CPU path'):
            call()
