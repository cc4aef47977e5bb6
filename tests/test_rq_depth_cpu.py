"""CPU tests of the residual quantiser at depth D > 1: the oracle (oracle/rq_oracle.py) against the reference's own
outputs (tests/golden/rq_*.pt, `python -m oracle.make_rq_golden`), the state dict against the reference module's
(names, shapes, dtypes, which keys alias one tensor), and the host-side argument checks of the D-aware methods."""
import json
import os

import pytest
import torch

from conftest import ROOT, golden_sample, load_golden

CODEC = {'d2_separate': ('rq_tdcrqvae3_d2_separate_b1_64_seed53.pt', 2, False),
         'd4_shared': ('rq_tdcrqvae3_d4_shared_b1_64_seed55.pt', 4, True)}


def net(network_g, depth, shared):
    g = dict(network_g)
    g.pop('type', None)
    g['code_shape'] = [32, 32, depth]
    g['shared_codebook'] = shared
    return g


def synth_codebooks(network_g, depth, shared):
    from oracle import rq_oracle
    from pgtformer_b200.spec import build_spec
    from pgtformer_b200.weights import synth_state_dict
    _, spec = build_spec(net(network_g, depth, shared))
    return rq_oracle.codebooks(synth_state_dict(spec, 0), depth)


def test_oracle_matches_the_reference_rq_bottleneck():
    from oracle import rq_oracle
    from oracle.make_rq_golden import rq_inputs
    g = load_golden('rq_bottleneck_T4096_K1024_E512_D4_seed41.pt')
    z, cbs = rq_inputs(g['T'], g['K'], g['E'], g['D'], g['seed'])
    quant_list, codes, _ = rq_oracle.quantize(cbs, z)
    assert torch.equal(codes, g['codes'])
    for d, q in enumerate(quant_list):
        s = golden_sample(q, g, 'quant_%d' % d)
        assert ((s - g['quant_%d' % d]).abs().max() / g['quant_%d_absmax' % d]).item() < 2e-5


@pytest.mark.parametrize('name', list(CODEC))
def test_oracle_matches_the_reference_codec_quantiser(network_g, name):
    from oracle import rq_oracle
    fixture, D, shared = CODEC[name]
    g = load_golden(fixture)
    cbs = synth_codebooks(network_g, D, shared)
    quant_list, codes, loss = rq_oracle.quantize(cbs, g['z_e'])
    assert torch.equal(codes, g['codes'])
    assert ((quant_list[-1] - g['z_q']).abs().max() / g['z_q'].abs().max()).item() < 2e-5
    assert abs(loss.item() - g['loss'].item()) <= 2e-5 * g['loss'].item()
    emb = rq_oracle.embed_with_depth(cbs, g['code'])
    assert torch.equal(golden_sample(emb, g, 'emb_with_depth'), g['emb_with_depth'])
    assert torch.equal(rq_oracle.embed_partial(cbs, g['code'], D - 1, 'add'), rq_oracle.embed_code(cbs, g['code']))
    for i, temp in enumerate(g['temps']):
        p, c = rq_oracle.soft_codes(cbs, g['z_e'], temp)
        assert torch.equal(c, g['soft_code_codes'][i])
        s = golden_sample(p, g, 'soft_code_%d' % i)
        assert (s - g['soft_code_%d' % i]).abs().max().item() < 2e-5


# --------------------------------------------------------------------------- state dict
def _specs():
    with open(os.path.join(ROOT, 'tests', 'golden', 'rq_state_dict_specs.json')) as f:
        return json.load(f)


@pytest.mark.parametrize('name,depth,shared', [('pgtformer_d2_separate', 2, False), ('pgtformer_d4_shared', 4, True),
                                               ('pgtformer_d2_shared', 2, True)])
def test_state_dict_matches_the_reference(network_g, name, depth, shared):
    from archs.pgtformer_arch import PGTFormer
    ref = _specs()[name]
    m = PGTFormer(**net(network_g, depth, shared))
    sd = m.state_dict()
    got = [[k, list(v.shape), str(v.dtype).replace('torch.', '')] for k, v in sd.items()]
    assert sorted(got) == sorted(ref['keys'])                  # strict loading is by name, not by order
    groups = {}
    for k, v in sd.items():
        groups.setdefault(v.data_ptr(), []).append(k)
    assert sorted(g for g in groups.values() if len(g) > 1) == sorted(ref['aliases'])
    assert m.quantizer_depth == depth and m.codebook_size == 1024
    m.load_state_dict(sd, strict=True)


def test_shared_codebook_load_keeps_the_last_copy(network_g):
    """The reference loads each aliased key into the one tensor in turn, so the last one wins."""
    from archs.pgtformer_arch import TDCRQVAE3
    g = net(network_g, 3, True)
    g.pop('dim_embd', None)
    m = TDCRQVAE3(**g)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    for d in range(3):
        sd['quantizer.codebooks.%d.weight' % d].fill_(float(d))
    m.load_state_dict(sd, strict=True)
    cbs = m.quantizer.codebooks
    assert all(cbs._modules[str(d)] is cbs._modules['0'] for d in range(3))
    assert (m.state_dict()['quantizer.codebooks.0.weight'] == 2.0).all()


def test_separate_codebooks_are_distinct(network_g):
    from archs.pgtformer_arch import TDCRQVAE3
    m = TDCRQVAE3(**net(network_g, 2, False))
    sd = m.state_dict()
    a, b = sd['quantizer.codebooks.0.weight'], sd['quantizer.codebooks.1.weight']
    assert a.data_ptr() != b.data_ptr() and not torch.equal(a, b)
    assert torch.equal(sd['quantizer.codebooks.1.embed_ema'], b[:-1])


# --------------------------------------------------------------------------- host-side argument checks
@pytest.fixture(scope='module')
def deep_model(network_g):
    from archs.pgtformer_arch import TDCRQVAE3
    return TDCRQVAE3(**net(network_g, 2, False))


@pytest.mark.parametrize('shape', [(3, 4, 4, 1), (3, 4, 4, 3), (3, 4, 4)])
def test_wrong_code_depth_is_a_value_error(deep_model, shape):
    code = torch.zeros(*shape, dtype=torch.int64)
    for call in (deep_model.decode_code, deep_model.get_code_emb_with_depth,
                 lambda c: deep_model.decode_partial_code(c, 0)):
        with pytest.raises(ValueError):
            call(code)


def test_partial_code_arguments(deep_model):
    code = torch.zeros(3, 4, 4, 2, dtype=torch.int64)
    with pytest.raises(AssertionError):
        deep_model.decode_partial_code(code, 2)
    with pytest.raises(NotImplementedError):
        deep_model.decode_partial_code(code, 1, decode_type='mean')
    with pytest.raises(ValueError):
        deep_model.decode_partial_code(code, -1)
    code[0, 0, 0, 1] = 1025
    with pytest.raises(IndexError):
        deep_model.decode_partial_code(code, 0)
    code[0, 0, 0, 1] = 1024                                    # the padding row is valid: the checks pass
    for d in (0, 1):
        with pytest.raises(RuntimeError, match='no CPU path'):
            deep_model.decode_partial_code(code, d, 'select')


def test_depth_zero_is_rejected(network_g):
    from archs.pgtformer_arch import TDCRQVAE3
    with pytest.raises(ValueError):
        TDCRQVAE3(**net(network_g, 0, True))
