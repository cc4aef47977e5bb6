"""TDRQVAE without a GPU: the oracle restatement (oracle/tdrqvae_oracle.py) against the reference's own outputs
(tests/golden/tdrqvae_ref_*.pt, oracle/make_tdrqvae_golden.py), the state-dict layout against the reference module's,
the registry, and the host-side checks that must fail before any CUDA work."""
import json
import os

import pytest
import torch

from conftest import ROOT, golden_sample, load_golden

SMALL = [('tdrqvae_ref_b1_t3_64_seed31.pt'), ('tdrqvae_ref_b2_t7_128_seed32.pt'), ('tdrqvae_ref_b1_t3_64x192_seed34.pt')]


@pytest.fixture(scope='module')
def tdrq_g(network_g):
    g = dict(network_g)
    g['type'] = 'TDRQVAE'
    return g


@pytest.fixture(scope='module')
def tdrq_spec(tdrq_g):
    from pgtformer_b200.spec import build_tdrqvae_spec
    return build_tdrqvae_spec(tdrq_g)


@pytest.fixture(scope='module')
def tdrq_sd(tdrq_spec):
    from pgtformer_b200.weights import synth_state_dict
    return synth_state_dict(tdrq_spec[1], 0)


@pytest.fixture(scope='module')
def model(tdrq_g):
    from pgtformer_b200.registry import ARCH_REGISTRY
    import archs  # noqa: F401
    return ARCH_REGISTRY.get('TDRQVAE')(**tdrq_g)


def _cmp(got, g, key):
    """max|got - ref| / max|ref| over what the fixture keeps of `key` (whole tensor or strided sample); latents may be
    given as [b*t, h, w, E] for the reference's [b, t, h, w, E]."""
    shape = g.get(key + '_shape', tuple(g[key].shape))
    assert got.numel() == torch.Size(shape).numel(), (key, got.shape, shape)
    got = got.reshape(shape)
    if key + '_stride' in g:
        s = golden_sample(got, g, key)
        return ((s - g[key].float()).abs().max() / g[key + '_absmax']).item()
    ref = g[key].float()
    return ((got.float().cpu() - ref).abs().max() / ref.abs().max()).item()


@pytest.mark.parametrize('name', SMALL)
def test_oracle_matches_reference_golden(name, tdrq_spec, tdrq_sd):
    from oracle import tdrqvae_oracle as O
    from oracle.make_tdrqvae_golden import golden_clips
    arch = tdrq_spec[0]
    g = load_golden(name)
    b, t, H, W = g['b'], g['t'], g['H'], g.get('W', g['H'])
    x = golden_clips(g['seed'], b, t, H, W)
    with torch.no_grad():
        (out, loss, code), lat = O.forward(tdrq_sd, arch, x, return_latents=True)
        z_q = O.forward(tdrq_sd, arch, x, code_only=True)[0]
        out_code = O.decode_code(tdrq_sd, arch, code.view(b * t, H // 16, W // 16, 1))
        soft, soft_code = O.get_soft_codes(tdrq_sd, arch, x.view(b * t, 3, H, W), 1.0)
    errs = {k: _cmp(v, g, k) for k, v in (('z_e', lat['z_e']), ('z_pre', lat['z_pre']), ('z_q', z_q), ('out', out),
                                          ('out_code', out_code), ('soft', soft))}
    print(name, errs)
    assert max(errs.values()) < 2e-5, errs
    assert torch.equal(code, g['codes'].long()) and torch.equal(soft_code, g['soft_codes'].long())
    assert abs(loss.item() - g['quant_loss'].item()) <= 2e-5 * g['quant_loss'].item()
    top2 = lat['dist'].topk(2, dim=-1, largest=False).values
    assert torch.allclose(top2[..., 1] - top2[..., 0], g['margin'].view(top2.shape[:-1]), rtol=1e-3, atol=1e-3)


def test_golden_files_are_small():
    for f in os.listdir(os.path.join(ROOT, 'tests', 'golden')):
        if f.startswith('tdrqvae_'):
            assert os.path.getsize(os.path.join(ROOT, 'tests', 'golden', f)) < 1_000_000, f


def test_state_dict_spec_is_the_references(model, tdrq_spec):
    """Names, shapes and dtypes of the reference module's state dict (oracle/make_tdrqvae_golden.py), the 125 x 125 int64
    relative_position_index buffers of tdswin_* included; a reference-named dict loads with strict=True."""
    with open(os.path.join(ROOT, 'tests', 'golden', 'tdrqvae_state_dict_spec.json')) as f:
        ref = json.load(f)
    ours = model.state_dict()
    assert len(ref) == 413 and set(ours) == set(ref)
    for k, (shape, dtype) in ref.items():
        assert list(ours[k].shape) == shape and str(ours[k].dtype) == dtype, k
    assert {k: (list(v[0]), 'torch.' + v[2]) for k, v in tdrq_spec[1].items()} == {k: tuple(v) for k, v in ref.items()}
    idx = ours['tdswin_post.blocks.3.attn.relative_position_index']
    assert idx.shape == (125, 125) and idx.dtype == torch.int64
    from oracle.swin3d_oracle import relative_position_index
    assert torch.equal(idx, relative_position_index((5, 5, 5)))
    sd = {k: torch.randn(v.shape) if v.dtype.is_floating_point else v.clone() for k, v in ours.items()}
    model.load_state_dict(sd, strict=True)
    assert torch.equal(model.state_dict()['encoder.mid.attn_1.q.weight'], sd['encoder.mid.attn_1.q.weight'])
    with pytest.raises(RuntimeError):
        model.load_state_dict({k: v for k, v in sd.items() if 'relative_position_index' not in k}, strict=True)


def test_registry_and_exports(tdrq_g):
    from pgtformer_b200.registry import ARCH_REGISTRY
    from archs import TDRQVAE
    from archs.tdrqvae_arch import TDRQVAE as T2
    assert ARCH_REGISTRY.get('TDRQVAE') is TDRQVAE is T2
    m = TDRQVAE(**tdrq_g)
    assert m.eval() is m and m.t == 3 and m.code_shape == [32, 32, 1]
    g = {k: v for k, v in tdrq_g.items() if k != 'tf'}
    assert TDRQVAE(**g).t == 7                                   # the reference's default, never read by forward
    with pytest.raises(RuntimeError, match='no CPU path'):
        m.engine()


def _bad(tdrq_g, **dd):
    g = dict(tdrq_g)
    top = {k: dd.pop(k) for k in list(dd) if k in ('code_shape', 'latent_shape', 'bottleneck_type', 'embed_dim')}
    g.update(top)
    g['ddconfig'] = dict(g['ddconfig'], **dd)
    return g


@pytest.mark.parametrize('bad', [
    dict(ch_mult=[1, 2, 4, 6, 8]),                     # AttnBlock of width 384 at the 64^2 level
    dict(attn_resolutions=[256]),                      # AttnBlock of width 128
    dict(num_head=4),                                  # Swin head width 128
    dict(num_head=64),                                 # Swin head width 8
    dict(window_size=[6, 5, 5]),                       # 150 tokens per window
    dict(code_shape=[32, 32, 2]),                      # quantiser depth 2
    dict(bottleneck_type='vq'),
    dict(double_z=True),
])
def test_constructor_rejects_what_the_kernels_cannot_run(tdrq_g, bad):
    from archs.tdrqvae_arch import TDRQVAE
    with pytest.raises(ValueError):
        TDRQVAE(**_bad(tdrq_g, **bad))


@pytest.mark.parametrize('ok', [dict(num_head=32), dict(num_head=16), dict(window_size=[2, 8, 8]),
                                dict(attn_resolutions=[32])])
def test_constructor_accepts_covered_variants(tdrq_g, ok):
    from archs.tdrqvae_arch import TDRQVAE
    TDRQVAE(**_bad(tdrq_g, **ok))


@pytest.mark.parametrize('key', ['latent_shape', 'code_shape', 'shared_codebook', 'restart_unused_codes'])
def test_missing_quantiser_keyword_is_a_keyerror(tdrq_g, key):
    from archs.tdrqvae_arch import TDRQVAE
    g = {k: v for k, v in tdrq_g.items() if k != key}
    with pytest.raises(KeyError):
        TDRQVAE(**g)


def test_argument_checks_raise_before_any_cuda_work(model):
    """On a CPU model the engine would raise RuntimeError ('no CPU path'): these must fail earlier, on the host."""
    x5 = torch.rand(1, 3, 3, 64, 64)
    for bad in (torch.rand(3, 3, 64, 64), torch.rand(1, 3, 3, 64, 96), torch.rand(1, 3, 4, 64, 64),
                torch.rand(0, 3, 3, 64, 64), torch.rand(1, 0, 3, 64, 64), 'clip'):
        for fn in (model, model.get_codes, model.get_codesbt):
            with pytest.raises(ValueError):
                fn(bad)
    for bad in (x5, torch.rand(3, 3, 64, 32), torch.rand(0, 3, 64, 64)):
        with pytest.raises(ValueError):
            model.encode(bad)
        with pytest.raises(ValueError):
            model.get_soft_codes(bad)
    for temp in (0.0, -1.0, float('nan'), float('inf'), 'warm'):
        with pytest.raises(ValueError):
            model.get_soft_codes(torch.rand(3, 3, 64, 64), temp)
    for bad in (torch.rand(3, 4, 4, 256), torch.rand(3, 4, 6, 512), torch.rand(3, 4, 4, 512).long(), torch.rand(4, 4, 512)):
        with pytest.raises(ValueError):
            model.decode(bad)
    for bad in (torch.zeros(3, 4, 4, 2, dtype=torch.long), torch.zeros(3, 4, 4, 1), torch.zeros(3, 4, 5, 1, dtype=torch.long),
                torch.zeros(1, 3, 4, 4, 1, dtype=torch.long)):
        with pytest.raises(ValueError):
            model.decode_code(bad)
    for v in (-1, 1025):
        code = torch.zeros(3, 4, 4, 1, dtype=torch.long)
        code[1, 2, 3, 0] = v
        with pytest.raises(IndexError):
            model.decode_code(code)
        with pytest.raises(IndexError):
            model.get_code_emb_with_depth(code)
    assert not hasattr(model, 'forward_partial_code')
