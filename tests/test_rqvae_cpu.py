"""RQVAE without a GPU: the oracle restatement (oracle/rqvae_oracle.py) against the reference's own outputs
(tests/golden/rqvae_*.pt, oracle/make_rqvae_golden.py), the state-dict layout against the reference module's, the
registry, the configurations the constructor rejects and the host-side checks that must fail before any CUDA work."""
import copy
import json
import os

import pytest
import torch

from conftest import ROOT, golden_sample, load_golden

FIXTURES = ['rqvae_r1_b1_256x256_seed81.pt', 'rqvae_r1_b2_256x256_seed82.pt', 'rqvae_r2_b2_128x128_seed83.pt',
            'rqvae_r2_b1_128x256_seed84.pt']


def config(name):
    from oracle.make_rqvae_golden import CONFIGS
    return copy.deepcopy(CONFIGS[name])


def build(g):
    from archs.rqvae_arch import RQVAE
    return RQVAE(**g)


@pytest.fixture(scope='module')
def models():
    return {c: build(config(c)) for c in ('r1', 'r2')}


def _err(got, g, key):
    s = golden_sample(got, g, key)
    return ((s - g[key].float()).abs().max() / g[key + '_absmax']).item()


@pytest.mark.parametrize('name', FIXTURES)
def test_oracle_matches_reference_golden(name, models):
    from oracle import rqvae_oracle as O
    from oracle.make_rqvae_golden import golden_images
    g = load_golden(name)
    m = models[g['config']]
    sd = {k: v.double() if v.dtype.is_floating_point else v for k, v in m.state_dict().items()}
    x = golden_images(g['seed'], g['b'], g['H'], g['W']).double()
    with torch.no_grad():
        out, loss, code = O.forward(sd, m.arch, x)
        z_q = O.forward(sd, m.arch, x, code_only=True)[0]
        z_e = O.encode(sd, m.arch, x)
        ref_code = g['codes'].long()
        errs = {'out': _err(out, g, 'out'), 'z_q': _err(z_q, g, 'z_q'), 'z_e': _err(z_e, g, 'z_e'),
                'out_code': _err(O.decode_code(sd, m.arch, ref_code), g, 'out_code'),
                'out_select1': _err(O.decode_partial_code(sd, m.arch, ref_code, 1, 'select'), g, 'out_select1'),
                'out_add1': _err(O.decode_partial_code(sd, m.arch, ref_code, 1, 'add'), g, 'out_add1')}
        if 'soft' in g:
            soft, soft_code = O.get_soft_codes(sd, m.arch, x, 1.0)
            errs['soft'] = _err(soft, g, 'soft')
            assert torch.equal(soft_code, ref_code)
    print(name, errs)
    assert max(errs.values()) < 2e-5, errs
    # fp64 against the reference's fp32: a code may differ only where the reference's own margin is at rounding level
    differ = code != ref_code
    assert (g['margin'][differ] < 1e-3).all(), g['margin'][differ]
    assert abs(loss.item() - g['quant_loss'].item()) <= 1e-4 * g['quant_loss'].item()


def test_golden_files_are_small():
    for f in os.listdir(os.path.join(ROOT, 'tests', 'golden')):
        if f.startswith('rqvae_'):
            assert os.path.getsize(os.path.join(ROOT, 'tests', 'golden', f)) < 1_000_000, f


@pytest.mark.parametrize('cfg,entries', [('r1', 398), ('r2', 307)])
def test_state_dict_spec_is_the_references(models, cfg, entries):
    """Names, shapes and dtypes of the reference module's state dict (oracle/make_rqvae_golden.py): R1 with a shared
    codebook listed under all four depths, R2 with per-depth codebooks of 512, 1024 and 256 codes; a reference-named
    dict loads with strict=True."""
    from pgtformer_b200.spec import build_rqvae_spec
    with open(os.path.join(ROOT, 'tests', 'golden', 'rqvae_%s_state_dict_spec.json' % cfg)) as f:
        ref = json.load(f)
    m = models[cfg]
    ours = m.state_dict()
    assert len(ref) == entries and set(ours) == set(ref)
    for k, (shape, dtype) in ref.items():
        assert list(ours[k].shape) == shape and str(ours[k].dtype) == dtype, k
    spec = build_rqvae_spec(config(cfg))[1]
    assert {k: (list(v[0]), 'torch.' + v[2]) for k, v in spec.items()} == {k: tuple(v) for k, v in ref.items()}
    sd = {k: torch.randn(v.shape) for k, v in ours.items()}
    if cfg == 'r1':                                         # one shared VQEmbedding: every depth's keys are one tensor
        for d in (1, 2, 3):
            for leaf in ('weight', 'cluster_size_ema', 'embed_ema'):
                sd['quantizer.codebooks.%d.%s' % (d, leaf)] = sd['quantizer.codebooks.0.%s' % leaf]
    m2 = build(config(cfg))
    m2.load_state_dict(sd, strict=True)
    assert torch.equal(m2.state_dict()['decoder.conv_out.weight'], sd['decoder.conv_out.weight'])
    with pytest.raises(RuntimeError):
        m2.load_state_dict({k: v for k, v in sd.items() if k != 'quant_conv.bias'}, strict=True)


def test_registry_and_exports():
    from pgtformer_b200.registry import ARCH_REGISTRY
    from archs import RQVAE
    from archs.rqvae_arch import RQVAE as R2
    assert ARCH_REGISTRY.get('RQVAE') is RQVAE is R2
    m = RQVAE(**config('r1'))
    assert m.eval() is m and m.code_shape == [8, 8, 4]
    with pytest.raises(RuntimeError, match='no CPU path'):
        m.engine()


def _bad(name, **kw):
    g = config(name)
    for k in list(kw):
        if k in g['ddconfig'] or k in ('resamp_with_conv', 'give_pre_end'):
            g['ddconfig'][k] = kw.pop(k)
    g.update(kw)
    return g


@pytest.mark.parametrize('bad', [
    dict(ch=96, ch_mult=[1, 1, 2, 2, 4, 4]),           # stem width 96
    dict(ch=256, ch_mult=[1, 1, 1, 1, 2, 2]),          # stem width 256
    dict(in_channels=4),
    dict(double_z=True),
    dict(resamp_with_conv=False),
    dict(give_pre_end=True),
    dict(attn_resolutions=[128]),                      # AttnBlock of width 128 at 128^2
    dict(code_shape=[4, 4, 4]),                        # code-shape divisor 2
    dict(latent_shape=[8, 8, 128]),                    # codebook width != embed_dim
    dict(embed_dim=192, latent_shape=[8, 8, 192]),     # codebook width not a multiple of 128
    dict(embed_dim=640, latent_shape=[8, 8, 640]),     # codebook width > 512
    dict(n_embed=2000),                                # K not a multiple of 128
    dict(n_embed=[2048] * 4),                          # a list with a shared codebook (the reference raises too)
    dict(bottleneck_type='vq'),
])
def test_constructor_rejects_what_the_kernels_cannot_run(bad):
    with pytest.raises(ValueError):
        build(_bad('r1', **bad))


def test_constructor_accepts_covered_variants():
    build(_bad('r1', attn_resolutions=[16, 8]))        # AttnBlocks of widths 512 and 512
    build(_bad('r1', attn_resolutions=[32]))           # width 256
    build(_bad('r2', n_embed=384, shared_codebook=True))


def test_constructor_rejects_bad_per_depth_lists():
    with pytest.raises(ValueError):
        build(_bad('r2', n_embed=[512, 1024]))         # two sizes for depth 3
    with pytest.raises(ValueError):
        build(_bad('r2', n_embed=[512, 1000, 256]))    # K not a multiple of 128


@pytest.mark.parametrize('key', ['latent_shape', 'code_shape', 'shared_codebook', 'restart_unused_codes'])
def test_missing_quantiser_keyword_is_a_keyerror(key):
    g = {k: v for k, v in config('r2').items() if k != key}
    with pytest.raises(KeyError):
        build(g)


def test_argument_checks_raise_before_any_cuda_work(models):
    """On a CPU model the engine would raise RuntimeError ('no CPU path'): these must fail earlier, on the host."""
    m = models['r2']                                   # f = 8: images multiples of 32
    for bad in (torch.rand(1, 1, 3, 64, 64), torch.rand(1, 3, 64, 48), torch.rand(1, 4, 64, 64), torch.rand(0, 3, 64, 64),
                torch.rand(2, 3, 64, 64).long(), 'image'):
        for fn in (m, m.get_codes, m.encode, m.get_soft_codes, lambda x: m.forward_partial_code(x, 0)):
            with pytest.raises(ValueError):
                fn(bad)
    for bad in (torch.rand(2, 3, 64, 64), torch.rand(1, 2, 3, 64, 48)):
        with pytest.raises(ValueError):
            m.get_codesbt(bad)
    with pytest.raises(ValueError, match='one size'):
        m.get_soft_codes(torch.rand(1, 3, 64, 64))     # codebooks of 512, 1024 and 256 codes
    for temp in (0.0, -1.0, float('nan'), 'warm'):
        with pytest.raises(ValueError):
            models['r1'].get_soft_codes(torch.rand(1, 3, 128, 128), temp)
    for bad in (torch.rand(2, 4, 4, 256), torch.rand(2, 4, 6, 128), torch.rand(2, 4, 4, 128).long()):
        with pytest.raises(ValueError):
            m.decode(bad)
    for bad in (torch.zeros(2, 4, 4, 2, dtype=torch.long), torch.zeros(2, 4, 4, 3), torch.zeros(2, 4, 5, 3, dtype=torch.long)):
        with pytest.raises(ValueError):
            m.decode_code(bad)
    for d, v in ((0, 513), (1, 1025), (2, 257), (2, -1)):
        code = torch.zeros(2, 4, 4, 3, dtype=torch.long)
        code[1, 2, 3, d] = v
        for fn in (m.decode_code, m.get_code_emb_with_depth, lambda c: m.decode_partial_code(c, 2, 'add')):
            with pytest.raises(IndexError):
                fn(code)
    code = torch.zeros(2, 4, 4, 3, dtype=torch.long)
    code[..., 1] = 1024                                # depth 1's padding row is in range
    with pytest.raises(NotImplementedError):
        m.decode_partial_code(code, 1, 'mean')
