"""TDRQVAE on the H100 through the C ABI: the engine's AttnBlock and the Video-Swin layers against the oracle
(oracle/tdrqvae_oracle.py, oracle/swin3d_oracle.py) on identical bf16 inputs, the model methods against the reference's
own outputs (tests/golden/tdrqvae_ref_*.pt) and the identities between the methods.

Bounds: a block (GroupNorm, two bf16 GEMMs and the flash-style core with one bf16 rounding of P) 1.5e-2 * max|ref|, the
lower end of DESIGN §2's block bound; the Video-Swin layer 2e-2 * max|ref| as in test_swin3d_gpu.py; the model methods
those of test_codec_gpu.py (encode 2.5e-2 * max|ref|, frames PSNR > 35 dB and 8e-2 * max|ref|)."""
import math

import pytest
import torch

from conftest import golden_sample, load_golden
from oracle import swin3d_oracle as S
from oracle import tdrqvae_oracle as O
from test_swin3d_gpu import test_window3d_attention_core as window3d_core

pytestmark = pytest.mark.gpu
DEV = 'cuda'
FIXTURES = ['tdrqvae_ref_b1_t3_64_seed31.pt', 'tdrqvae_ref_b2_t7_128_seed32.pt', 'tdrqvae_ref_b1_t3_512_seed33.pt',
            'tdrqvae_ref_b1_t3_64x192_seed34.pt']


@pytest.fixture(scope='module')
def tdrq_g(network_g):
    g = dict(network_g)
    g['type'] = 'TDRQVAE'
    return g


@pytest.fixture(scope='module')
def model(tdrq_g):
    from pgtformer_b200.registry import ARCH_REGISTRY
    import archs  # noqa: F401
    return ARCH_REGISTRY.get('TDRQVAE')(**tdrq_g).to(DEV).eval()


@pytest.fixture(scope='module')
def sd64(model):
    return {k: v.double() if v.dtype.is_floating_point else v for k, v in model.state_dict().items()}


@pytest.fixture(scope='module')
def sd64_cpu(sd64):
    """The fp64 weights on the host: the Video-Swin oracle builds its shift mask on the CPU."""
    return {k: v.cpu() for k, v in sd64.items()}


def relerr(got, ref):
    got, ref = got.double().cpu(), ref.double().cpu()
    assert got.shape == ref.shape, (got.shape, ref.shape)
    assert torch.isfinite(got).all()
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-12)).item()


def psnr(got, ref):
    mse = (got.float().cpu() - ref.float().cpu()).pow(2).mean().item()
    return 99.0 if mse == 0 else 10 * math.log10(1.0 / mse)


# --------------------------------------------------------------------------- blocks vs the oracle
@pytest.mark.parametrize('p,Fr,H,W', [
    ('encoder.down.2.attn.0', 2, 128, 128),            # C = 256, L = 16384
    ('decoder.up.3.attn.1', 3, 64, 64),                # C = 256, L = 4096
    ('encoder.mid.attn_1', 3, 32, 32),                 # C = 512, L = 1024
    ('decoder.up.2.attn.1', 2, 30, 26),                # C = 256, ragged L = 780
    ('decoder.mid.attn_1', 2, 9, 7),                   # C = 512, ragged L = 63
])
def test_attn_block_against_oracle(model, sd64, p, Fr, H, W):
    eng = model.engine()
    C = sd64[p + '.q.weight'].shape[0]
    x = torch.randn(Fr, H, W, C, generator=torch.Generator().manual_seed(Fr * H + W)).to(DEV).bfloat16()
    y = eng.attn_block(x, p)
    ref = O.attn_block(sd64, p, x.double().permute(0, 3, 1, 2)).permute(0, 2, 3, 1)
    e = relerr(y, ref)
    print('%s (C %d, L %d): %.3e of max|ref| %.2f' % (p, C, H * W, e, ref.abs().max().item()))
    assert y.dtype == torch.bfloat16 and e < 1.5e-2


@pytest.mark.parametrize('B,D,shift', [(1, 3, (2, 2, 2)), (1, 7, (2, 2, 2)), (2, 7, (0, 0, 0))])
def test_window3d_core_d64_n125(B, D, shift):
    """The never-before-run launch of tdswin_*: head width 64, up to 125 tokens (D >= 5) per window, 55 KB of dynamic
    shared memory."""
    window3d_core(B, D, 32, 32, 512, 8, (5, 5, 5), shift, False)


@pytest.mark.parametrize('D', [3, 7])
def test_basic_layer_512_against_oracle(D):
    from modules.swin import BasicLayer
    layer = BasicLayer(512, 4, 8, (5, 5, 5))
    sd = S.synth_state(layer.state_dict(), 40 + D)
    layer.load_state_dict(sd, strict=True)
    layer = layer.to(DEV)
    x = torch.randn(1, 512, D, 32, 32, generator=torch.Generator().manual_seed(D))
    y = layer(x.to(DEV))
    sdd = {k: v.double() if v.dtype.is_floating_point else v for k, v in sd.items()}
    ref = S.basic_layer(sdd, '', x.double(), 4, 8, (5, 5, 5))
    e = relerr(y, ref)
    print('BasicLayer(512, 4, 8, (5,5,5)) D=%d: %.3e of max|ref| %.2f' % (D, e, ref.abs().max().item()))
    assert e < 2e-2


def test_engine_swin_rows_equal_the_module(model):
    """tdswin_pre of the engine and modules.swin.BasicLayer with the same weights run the same launches: equal bits."""
    from modules.swin import BasicLayer
    eng = model.engine()
    layer = BasicLayer(512, 4, 8, (5, 5, 5))
    layer.load_state_dict({k[len('tdswin_pre.'):]: v for k, v in model.state_dict().items()
                           if k.startswith('tdswin_pre.')}, strict=True)
    layer = layer.to(DEV)
    b, t, h, w = 2, 6, 8, 12
    z = torch.randn(b * t * h * w, 512, generator=torch.Generator().manual_seed(3)).to(DEV).bfloat16()
    rows = eng.tdswin('tdswin_pre', z, b, t, h, w)
    ref = layer(z.float().view(b, t, h, w, 512).permute(0, 4, 1, 2, 3))
    assert torch.equal(rows.float().view(b, t, h, w, 512), ref.permute(0, 2, 3, 4, 1))


# --------------------------------------------------------------------------- the model vs the reference's outputs
def _take(t, g, key):
    """Our tensor in the fixture's form: the strided sample, or the whole tensor reshaped to the reference's shape."""
    if key + '_stride' in g:
        return golden_sample(t.reshape(g[key + '_shape']), g, key), g[key].float(), g[key + '_absmax']
    ref = g[key].float()
    return t.float().cpu().reshape(ref.shape), ref, ref.abs().max().item()


@pytest.mark.parametrize('name', FIXTURES)
def test_methods_against_reference_golden(model, name):
    from oracle.make_tdrqvae_golden import golden_clips
    g = load_golden(name)
    b, t, H, W = g['b'], g['t'], g['H'], g.get('W', g['H'])
    h, w = H // 16, W // 16
    x = golden_clips(g['seed'], b, t, H, W).to(DEV)
    eng = model.engine()
    z_e, z_pre = eng.latents(x)
    res = {}
    for key, v in (('z_e', z_e), ('z_pre', z_pre)):
        s, ref, amax = _take(v, g, key)
        res[key] = ((s - ref).abs().max() / amax).item()
    assert torch.equal(model.encode(x.view(b * t, 3, H, W)), z_e)
    out, loss, code = model(x)
    assert out.shape == (b, t, 3, H, W) and out.dtype == torch.float32 and code.shape == (b, t, h, w, 1)
    ref_code = g['codes'].long()
    agree = (code.cpu() == ref_code).float().mean().item()
    # codes must match wherever the reference's top-2 distance margin clearly exceeds the distance error our z error
    # causes: d_k = |z - e_k|^2 moves by about 2 <dz, z - e_k>, i.e. 2 rms(dz) |z - e_k| for an error uncorrelated with
    # z - e_k; "clearly" is 3x that, with |z - e_k| the token's distance to the reference's code
    s, ref, _ = _take(z_pre, g, 'z_pre')
    rms = (s - ref).pow(2).mean().sqrt().item()
    cb = model.quantizer.codebooks._modules['0'].weight.detach().float()
    reach = (z_pre.reshape(-1, 512) - cb[ref_code.reshape(-1).to(DEV)]).norm(dim=1).cpu()
    confident = g['margin'].reshape(-1) > 3 * 2 * rms * reach
    same_conf = (code.cpu().reshape(-1) == ref_code.reshape(-1))[confident].all().item()
    res.update(code_agree=agree, confident=confident.float().mean().item(),
               loss=abs(loss.item() - g['quant_loss'].item()) / g['quant_loss'].item())
    # teacher-forced: the reference's own codes into tdswin_post and the decoder
    out_tf, _, _ = eng.forward(x, force_codes=ref_code)
    zq_tf, _, _ = eng.forward(x, code_only=True, force_codes=ref_code)
    s, ref, amax = _take(out_tf, g, 'out')
    res.update(out_psnr=psnr(s, ref), out_err=((s - ref).abs().max() / amax).item())
    s, ref, amax = _take(zq_tf, g, 'z_q')
    res['z_q_err'] = ((s - ref).abs().max() / amax).item()
    out_code = model.decode_code(ref_code.view(b * t, h, w, 1))
    s, ref, amax = _take(out_code, g, 'out_code')
    res.update(out_code_psnr=psnr(s, ref), out_code_err=((s - ref).abs().max() / amax).item())
    soft, soft_code = model.get_soft_codes(x.view(b * t, 3, H, W), 1.0)
    res['soft_code_agree'] = (soft_code.cpu() == g['soft_codes'].long()).float().mean().item()
    print('%s: %s' % (name, res))
    assert res['z_e'] < 2.5e-2 and res['z_pre'] < 2.5e-2
    assert agree > 0.9 and same_conf and res['soft_code_agree'] > 0.9 and res['loss'] < 5e-2
    assert res['out_psnr'] > 35.0 and res['out_err'] < 8e-2 and res['z_q_err'] < 2.5e-2
    assert res['out_code_psnr'] > 35.0 and res['out_code_err'] < 8e-2


# --------------------------------------------------------------------------- identities
def test_batch_equals_per_clip(model):
    x = torch.rand(2, 3, 3, 64, 64, generator=torch.Generator().manual_seed(5)).to(DEV)
    out, loss, code = model(x)
    for i in range(2):
        o, _, c = model(x[i:i + 1])
        assert torch.equal(o, out[i:i + 1]) and torch.equal(c, code[i:i + 1])
    zq, loss2, code2 = model(x, code_only=True)
    assert zq.shape == (2, 3, 4, 4, 512) and zq.dtype == torch.float32
    assert torch.equal(code2, code) and torch.equal(loss2, loss)
    assert torch.equal(model(x[1:], code_only=True)[0], zq[1:])


@pytest.mark.parametrize('H,W', [(128, 64), (64, 192)])
@pytest.mark.parametrize('b,t', [(1, 1), (3, 2), (1, 5)])
def test_any_clip_length(model, sd64_cpu, b, t, H, W):
    """Any b, t >= 1 (t >= 5 fills the 5-frame window in depth); against the oracle with the same codes.  At 64 x 192
    the tile grids of several levels do not divide the frame."""
    x = torch.rand(b, t, 3, H, W, generator=torch.Generator().manual_seed(b * 10 + t)).to(DEV)
    out, loss, code = model(x)
    h, w = H // 16, W // 16
    assert out.shape == (b, t, 3, H, W) and code.shape == (b, t, h, w, 1)
    (ref, _, ref_code), lat = O.forward(sd64_cpu, model.arch, x.double().cpu(), force_codes=code.cpu().view(b * t, h, w, 1),
                                        return_latents=True)
    agree = (code.cpu() == ref_code).float().mean().item()
    print('b=%d t=%d: code agreement %.3f, out PSNR %.1f dB' % (b, t, agree, psnr(out, ref)))
    assert agree > 0.9 and psnr(out, ref) > 35.0 and relerr(out, ref) < 8e-2


def test_codes_and_decode_identities(model):
    x = torch.rand(2, 3, 3, 64, 64, generator=torch.Generator().manual_seed(7)).to(DEV)
    _, _, code = model(x)
    assert torch.equal(model.get_codes(x), code)
    assert torch.equal(model.get_codesbt(x), code.view(6, 4, 4, 1))
    c4 = code.view(6, 4, 4, 1)
    emb, none = model.get_code_emb_with_depth(c4)
    assert none is None and emb.shape == (6, 4, 4, 1, 512)
    out = model.decode_code(c4)
    assert out.shape == (6, 3, 64, 64) and torch.equal(out, model.decode(emb[..., 0, :]))
    assert torch.equal(model.decode_partial_code(c4, 0), out) and torch.equal(model.decode_partial_code(c4, 0, 'add'), out)


def test_get_soft_codes_is_the_kernel_on_encode(model):
    from pgtformer_b200 import ops
    x = torch.rand(4, 3, 64, 64, generator=torch.Generator().manual_seed(8)).to(DEV)
    cb = model.engine().w['codebook']
    p, code = model.get_soft_codes(x, 10.0)
    assert p.shape == (4, 4, 4, 1, 1024) and code.shape == (4, 4, 4, 1) and code.dtype == torch.int64
    z = model.encode(x).reshape(-1, 512)
    ref = torch.empty(z.shape[0], 1024, device=DEV)
    ops.soft_codes(z, cb, ops.codebook_pack(cb, 1024)[1], 1024, 10.0, ref)
    assert torch.equal(p.view(-1, 1024), ref)
    idx = torch.empty(z.shape[0], dtype=torch.int64, device=DEV)
    ops.l2_argmin_tc(z, cb, ops.codebook_pack(cb, 1024), 1024, idx)
    assert torch.equal(code.view(-1), idx)
    torch.manual_seed(3)
    _, s1 = model.get_soft_codes(x, 10.0, stochastic=True)
    torch.manual_seed(3)
    _, s2 = model.get_soft_codes(x, 10.0, stochastic=True)
    assert torch.equal(s1, s2) and s1.min() >= 0 and s1.max() < 1024


def test_other_models_unchanged_by_tdrqvae_calls(network_g, model):
    from archs.pgtformer_arch import PGTFormer, TDCRQVAE3
    opt = dict(network_g)
    opt.pop('type')
    pgt = PGTFormer(**opt).to(DEV).eval()
    vq = TDCRQVAE3(**opt).to(DEV).eval()
    x = torch.rand(3, 3, 64, 64, generator=torch.Generator().manual_seed(9)).to(DEV)
    a = [t.clone() for t in pgt(x, w=1, adain=True)]
    av = [t.clone() for t in vq(x)]
    model(torch.rand(1, 5, 3, 128, 128, generator=torch.Generator().manual_seed(10)).to(DEV))
    model.decode_code(torch.randint(0, 1025, (2, 4, 4, 1), generator=torch.Generator().manual_seed(11)))
    model.get_soft_codes(x, 1.0, stochastic=True)
    for u, v in zip(a, pgt(x, w=1, adain=True)):
        assert torch.equal(u, v)
    for u, v in zip(av, vq(x)):
        assert torch.equal(u, v)
