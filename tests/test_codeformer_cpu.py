"""VQAutoEncoder and CodeFormer without a GPU: the oracle restatement (oracle/vqgan_oracle.py) against the reference's own
outputs (tests/golden/vqgan_ref_*.pt, codeformer_ref_*.pt, oracle/make_codeformer_golden.py), the state-dict layouts
against the reference modules', the registry, the constructor rejections and the host-side checks that must fail before
any CUDA work."""
import json
import os

import pytest
import torch

from conftest import ROOT, golden_sample, load_golden

VQ_FIXTURES = ['vqgan_ref_b1_512x512_seed51.pt', 'vqgan_ref_b2_256x384_seed52.pt']
CF_FIXTURES = ['codeformer_ref_b1_512_seed61.pt', 'codeformer_ref_b2_512_seed62.pt']


@pytest.fixture(scope='module')
def vq_spec():
    from pgtformer_b200.spec import build_vqgan_spec
    return build_vqgan_spec({})


@pytest.fixture(scope='module')
def cf_spec():
    from pgtformer_b200.spec import build_codeformer_spec
    return build_codeformer_spec({})


def _sd(spec):
    from pgtformer_b200.weights import synth_state_dict
    return synth_state_dict(spec[1], 0)


def _err(t, g, key):
    return ((golden_sample(t, g, key) - g[key].float()).abs().max() / g[key + '_absmax']).item()


@pytest.mark.parametrize('name', VQ_FIXTURES)
def test_vqgan_oracle_matches_reference_golden(name, vq_spec):
    from oracle import vqgan_oracle as O
    from oracle.make_codeformer_golden import golden_images
    g = load_golden(name)
    x = golden_images(g['seed'], g['b'], g['H'], g['W'])
    sd = _sd(vq_spec)
    with torch.no_grad():
        out, loss, st, counts, z = O.vqgan_forward(sd, vq_spec[0], x)
        quant = O.vqgan_forward(sd, vq_spec[0], x, code_only=True)[0]
    errs = {'z': _err(z, g, 'z'), 'quant': _err(quant, g, 'quant'), 'out': _err(out, g, 'out')}
    print(name, errs)
    assert errs['z'] < 2e-5 and errs['quant'] < 2e-5 and errs['out'] < 2e-3      # out is stored as fp16
    assert torch.equal(st['min_encoding_indices'].view(-1), g['codes'].long())
    assert torch.equal(counts, g['usage'].int())
    for key, ref in (('loss', g['loss']), ('perplexity', g['perplexity']), ('mean_distance', g['mean_distance'])):
        v = loss if key == 'loss' else st[key]
        assert abs(v.item() - ref.item()) <= 2e-5 * abs(ref.item()), key
    assert torch.allclose(st['min_encoding_scores'].view(-1), g['scores'], rtol=2e-5, atol=0)


@pytest.mark.parametrize('name', CF_FIXTURES)
def test_codeformer_oracle_matches_reference_golden(name, cf_spec):
    from oracle import vqgan_oracle as O
    from oracle.make_codeformer_golden import golden_images
    g = load_golden(name)
    x = golden_images(g['seed'], g['b'], 512, 512)
    sd = _sd(cf_spec)
    with torch.no_grad():
        logits, lq = O.codeformer_forward(sd, cf_spec[0], x, code_only=True)
        errs = {'lq_feat': _err(lq, g, 'lq_feat'),
                'logits': ((logits.reshape(-1, logits.shape[-1])[g['logit_rows']] - g['logits_sel']).abs().max()
                           / g['logits_absmax']).item()}
        for i, (w, adain) in enumerate(g['cases']):
            out, logits2, _ = O.codeformer_forward(sd, cf_spec[0], x, w, adain)
            assert torch.equal(logits2, logits)
            errs['out%d' % i] = _err(out, g, 'out%d' % i)
    print(name, errs)
    assert errs['lq_feat'] < 2e-5 and errs['logits'] < 2e-5
    assert max(v for k, v in errs.items() if k.startswith('out')) < 2e-3          # out is stored as fp16
    codes = torch.topk(torch.softmax(logits, 2), 1, dim=2)[1].reshape(-1)
    assert torch.equal(codes, g['codes'].long())
    top2 = logits.reshape(-1, logits.shape[-1]).topk(2, dim=1).values
    assert torch.allclose(top2[:, 0] - top2[:, 1], g['margin'], rtol=1e-3, atol=1e-4)


def test_golden_files_are_small():
    for f in os.listdir(os.path.join(ROOT, 'tests', 'golden')):
        if f.startswith(('vqgan_', 'codeformer_')):
            assert os.path.getsize(os.path.join(ROOT, 'tests', 'golden', f)) < 1_000_000, f


@pytest.mark.parametrize('cls,spec_json,n', [('VQAutoEncoder', 'vqgan_state_dict_spec.json', 329),
                                             ('CodeFormer', 'codeformer_state_dict_spec.json', 515)])
def test_state_dict_spec_is_the_references(cls, spec_json, n):
    from pgtformer_b200.registry import ARCH_REGISTRY
    import archs  # noqa: F401
    model = ARCH_REGISTRY.get(cls)()
    with open(os.path.join(ROOT, 'tests', 'golden', spec_json)) as f:
        ref = json.load(f)
    ours = model.state_dict()
    assert len(ref) == n and list(ours) == list(ref)
    for k, (shape, dtype) in ref.items():
        assert list(ours[k].shape) == shape and str(ours[k].dtype) == dtype, k
    assert 'quantize.usage' not in ours
    usage = dict(model.named_buffers())['quantize.usage']
    assert usage.dtype == torch.int32 and usage.shape == (1024,) and int(usage.abs().sum()) == 0
    sd = {k: torch.randn(v.shape) for k, v in ours.items()}
    model.load_state_dict(sd, strict=True)
    assert torch.equal(model.state_dict()['quantize.embedding.weight'], sd['quantize.embedding.weight'])
    with pytest.raises(RuntimeError):
        model.load_state_dict({k: v for k, v in sd.items() if k != 'generator.blocks.8.conv.weight'}, strict=True)


def test_registry_and_exports():
    from pgtformer_b200.registry import ARCH_REGISTRY
    from archs import CodeFormer, VQAutoEncoder
    from archs.codeformer_arch import CodeFormer as C2
    from archs.vqgan_arch import VQAutoEncoder as V2
    assert ARCH_REGISTRY.get('VQAutoEncoder') is VQAutoEncoder is V2
    assert ARCH_REGISTRY.get('CodeFormer') is CodeFormer is C2
    assert issubclass(CodeFormer, VQAutoEncoder)
    m = CodeFormer(fix_modules=None, detach_16=False)
    assert m.eval() is m and m.w == 0 and m.adain is False and m.fix_modules is None
    with pytest.raises(RuntimeError, match='no CPU path'):
        m.engine()
    with pytest.raises(RuntimeError):
        m.train()


@pytest.mark.parametrize('cls,kw', [
    ('VQAutoEncoder', dict(quantizer='gumbel')),
    ('VQAutoEncoder', dict(nf=32)),
    ('VQAutoEncoder', dict(ch_mult=[1, 2, 2, 4, 4, 6])),          # AttnBlock width 384
    ('VQAutoEncoder', dict(attn_resolutions=[16, 256])),          # AttnBlock width 128
    ('VQAutoEncoder', dict(ch_mult=[1, 2, 2, 4, 4, 7])),          # a level width that is not a multiple of 32
    ('VQAutoEncoder', dict(last_silu=True)),
    ('CodeFormer', dict(quantizer='gumbel')),
    ('CodeFormer', dict(latent_size=64)),
    ('CodeFormer', dict(img_size=256, latent_size=256)),
    ('CodeFormer', dict(connect_list=['8'])),
    ('CodeFormer', dict(res_blocks=1)),                          # the fusion table's blocks are not at their sizes
])
def test_constructor_rejects_what_the_kernels_cannot_run(cls, kw):
    from pgtformer_b200.registry import ARCH_REGISTRY
    import archs  # noqa: F401
    with pytest.raises(ValueError):
        ARCH_REGISTRY.get(cls)(**kw)


@pytest.mark.parametrize('cls', ['VQAutoEncoder', 'CodeFormer'])
def test_unknown_keyword_is_a_typeerror(cls):
    from pgtformer_b200.registry import ARCH_REGISTRY
    import archs  # noqa: F401
    with pytest.raises(TypeError):
        ARCH_REGISTRY.get(cls)(foo=1)
    with pytest.raises(TypeError):
        ARCH_REGISTRY.get(cls)(dim_embd_typo=512)


def test_quantize_usage_methods():
    """reset_usage / get_usage live on `quantize`, as on the reference's VectorQuantizer."""
    from archs import VQAutoEncoder
    m = VQAutoEncoder()
    m.quantize.usage[:256] = 3
    assert abs(float(m.quantize.get_usage()) - 0.25) < 1e-7
    m.quantize.reset_usage()
    u = dict(m.named_buffers())['quantize.usage']
    assert u.dtype == torch.int32 and int(u.abs().sum()) == 0 and 'quantize.usage' not in m.state_dict()


def test_constructor_accepts_covered_variants():
    from archs import CodeFormer, VQAutoEncoder
    VQAutoEncoder(img_size=256)
    VQAutoEncoder(attn_resolutions=[16, 32])
    CodeFormer(connect_list=['32', '64'])


def test_argument_checks_raise_before_any_cuda_work():
    """On a CPU model the engine would raise RuntimeError ('no CPU path'): these must fail earlier, on the host."""
    from archs import CodeFormer, VQAutoEncoder
    vq, cf = VQAutoEncoder(), CodeFormer()
    for bad in (torch.rand(3, 512, 512), torch.rand(1, 4, 512, 512), torch.rand(0, 3, 512, 512),
                torch.rand(1, 3, 512, 500), torch.rand(1, 3, 64, 128), torch.zeros(1, 3, 256, 256, dtype=torch.long),
                'image'):
        with pytest.raises(ValueError):
            vq(bad)
        with pytest.raises(ValueError):
            cf(bad)
    for bad in (torch.rand(1, 3, 256, 256), torch.rand(1, 3, 512, 384), torch.rand(1, 3, 1024, 1024)):
        with pytest.raises(ValueError):
            cf(bad, w=0.5)
    with pytest.raises(IndexError):
        cf(torch.rand(1, 3, 512, 512), force_codes=torch.full((1, 256), 1024))


def test_model_path(tmp_path, vq_spec):
    from archs import VQAutoEncoder
    sd = {k: v * 0.5 if v.is_floating_point() else v for k, v in _sd(vq_spec).items()}
    for key in ('params_ema', 'params'):
        p = tmp_path / (key + '.pth')
        torch.save({key: sd, 'other': {}}, p)
        m = VQAutoEncoder(model_path=str(p))
        assert torch.equal(m.state_dict()['encoder.blocks.0.weight'], sd['encoder.blocks.0.weight'])
    p = tmp_path / 'both.pth'
    torch.save({'params_ema': sd, 'params': _sd(vq_spec)}, p)
    assert torch.equal(VQAutoEncoder(model_path=str(p)).state_dict()['quantize.embedding.weight'],
                       sd['quantize.embedding.weight'])
    p = tmp_path / 'bad.pth'
    torch.save({'state_dict': sd}, p)
    with pytest.raises(ValueError, match='Wrong params'):
        VQAutoEncoder(model_path=str(p))
