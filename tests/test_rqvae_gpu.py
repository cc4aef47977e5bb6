"""RQVAE on the H100 through the C ABI: the 128-wide RGB stem and decoder tail against fp64, the codebook-split argmin
against an fp64 argmin and the unsplit kernel (random and adversarial codebooks), the model methods against the
reference's own outputs (tests/golden/rqvae_*.pt) and the identities between the methods.

Bounds are those of test_tdrqvae_gpu.py (codes equal wherever the reference's top-2 margin exceeds the distance error
our latent error causes, decoded images PSNR > 35 dB), except encode: 2.5e-2 * max|ref| for the four-level R2 encoder,
3e-2 for the six-level R1 encoder, whose two extra levels of bf16 activations measure 2.4-2.6e-2."""
import copy
import math

import pytest
import torch
import torch.nn.functional as F

from conftest import golden_sample, load_golden

pytestmark = pytest.mark.gpu
DEV = 'cuda'
FIXTURES = ['rqvae_r1_b1_256x256_seed81.pt', 'rqvae_r1_b2_256x256_seed82.pt', 'rqvae_r2_b2_128x128_seed83.pt',
            'rqvae_r2_b1_128x256_seed84.pt']


def config(name):
    from oracle.make_rqvae_golden import CONFIGS
    return copy.deepcopy(CONFIGS[name])


@pytest.fixture(scope='module')
def models():
    from pgtformer_b200.registry import ARCH_REGISTRY
    import archs  # noqa: F401
    cls = ARCH_REGISTRY.get('RQVAE')
    return {c: cls(**config(c)).to(DEV).eval() for c in ('r1', 'r2')}


def psnr(got, ref):
    mse = (got.float().cpu() - ref.float().cpu()).pow(2).mean().item()
    return 99.0 if mse == 0 else 10 * math.log10(1.0 / mse)


# --------------------------------------------------------------------------- the 128-wide stem
@pytest.mark.parametrize('Fr,H,W', [(2, 64, 64), (1, 96, 160), (3, 40, 24)])
def test_rgb_stem_128_against_fp64(Fr, H, W):
    """encoder.conv_in at ch = 128 (3x3 / 1, Cin = 3): bf16 output against an fp64 conv of the same bf16-rounded
    weights; the GroupNorm(32) partial sums of its epilogue (when a frame is whole 128-row tiles) against fp64 sums."""
    from pgtformer_b200 import ops
    from pgtformer_b200.engine import _pack_rgb
    g = torch.Generator().manual_seed(Fr * 1000 + H + W)
    x = torch.rand(Fr, 3, H, W, generator=g)
    w = (torch.rand(128, 3, 3, 3, generator=g) * 2 - 1) / math.sqrt(27)
    b = (torch.rand(128, generator=g) * 2 - 1) * 0.05
    out = torch.empty(Fr, H, W, 128, dtype=torch.bfloat16, device=DEV)
    stats = None
    if (H * W) % 128 == 0:
        stats = torch.zeros(Fr * (H * W // 32) * 64, dtype=torch.float32, device=DEV)
    ops.conv_rgb(x.to(DEV), _pack_rgb(w.to(DEV)), b.to(DEV), out, 3, 1, 1, gn_stats=stats)
    torch.cuda.synchronize()
    wq = w.to(torch.bfloat16).double()
    xq = x.to(torch.bfloat16).double()
    ref = (F.conv2d(xq, wq, padding=1) + b.double()[None, :, None, None]).permute(0, 2, 3, 1)
    err = ((out.double().cpu() - ref).abs().max() / ref.abs().max()).item()
    print('stem 128 [%d, %d, %d]: %.2e of max|ref|' % (Fr, H, W, err))
    assert err < 8e-3
    if stats is not None:
        got = stats.view(Fr, -1, 32, 2).double().sum(1).cpu()
        r = ref.reshape(Fr, H * W, 32, 4)
        want = torch.stack([r.sum((1, 3)), r.pow(2).sum((1, 3))], -1)
        e = ((got - want).abs() / want.abs().clamp_min(1.0)).max().item()
        print('  GroupNorm sums: %.2e' % e)
        assert e < 1e-3


# --------------------------------------------------------------------------- the 128-wide decoder tail
@pytest.mark.parametrize('silu', [True, False])
@pytest.mark.parametrize('Fr,H,W', [(2, 32, 16), (1, 48, 40)])
def test_conv_out_128_against_fp64(silu, Fr, H, W):
    """decoder.norm_out (+ SiLU) + conv_out fused at Cin = 128 (two K-panels per pixel) against fp64 of the same bf16
    input, GroupNorm affine terms and bf16 weights; the kernel rounds the normalised activation to bf16 once."""
    from pgtformer_b200 import ops
    from pgtformer_b200.engine import _pack_conv
    g = torch.Generator().manual_seed(Fr * 100 + H + W + silu)
    x = (torch.randn(Fr, H, W, 128, generator=g) * 2 + 0.5).to(torch.bfloat16)
    gamma, beta = 1 + 0.1 * torch.randn(128, generator=g), 0.05 * torch.randn(128, generator=g)
    w = torch.randn(3, 128, 3, 3, generator=g) / math.sqrt(9 * 128)
    b = 0.05 * torch.randn(3, generator=g)
    xd = x.to(DEV)
    ab = ops.groupnorm_ab(xd, gamma.to(DEV), beta.to(DEV), torch.empty(Fr * 256, device=DEV))
    out = torch.empty(Fr, 3, H, W, device=DEV)
    assert ops.conv_out_gn(xd, ab, _pack_conv(w.to(DEV)), 3, b.to(DEV), out, silu=silu) is not None
    xr = x.double().permute(0, 3, 1, 2)
    y = F.group_norm(xr, 32, gamma.double(), beta.double(), eps=1e-6)
    y = F.silu(y) if silu else y
    ref = F.conv2d(y, w.to(torch.bfloat16).double(), b.double(), padding=1)
    err = ((out.double().cpu() - ref).abs().max() / ref.abs().max()).item()
    print('conv_out 128 silu=%d [%d, %d, %d]: %.2e of max|ref|' % (silu, Fr, H, W, err))
    assert err < 1.5e-2


# --------------------------------------------------------------------------- the codebook-split argmin
def _argmin64(z, cb, K):
    d = (z.double()[:, None, :] - cb.double()[None, :K, :]).pow(2).sum(-1) if z.shape[0] * K <= 1 << 22 else None
    if d is None:
        zz, c = z.double(), cb[:K].double()
        d = zz.pow(2).sum(1, keepdim=True) - 2 * zz @ c.t() + c.pow(2).sum(1)[None]
    return d.argmin(1)                                   # first index on ties


def _split_case(T, K, E, S, kind, seed):
    from pgtformer_b200 import ops
    g = torch.Generator().manual_seed(seed)
    cb = torch.randn(K + 1, E, generator=g)
    z = torch.randn(T, E, generator=g) * 0.9
    if kind == 'duplicates':                             # equal rows on both sides of every split boundary
        per = -(-(K // 128) // min(S, K // 128)) * 128
        for b in range(per, K, per):
            cb[b] = cb[b - 1]
            z[(b // per) % T] = cb[b] + 1e-3 * torch.randn(E, generator=g)
    elif kind == 'constant':                             # every row overflows to the exhaustive kernel
        cb[:] = cb[0]
    elif kind == 'equal_row':                            # z equal to a code row
        z[: min(T, 64)] = cb[torch.randint(0, K, (min(T, 64),), generator=g)]
    cbd, zd = cb.to(DEV), z.to(DEV)
    pack = ops.codebook_pack(cbd, K)
    got = torch.empty(T, dtype=torch.int64, device=DEV)
    q = torch.empty(T, E, device=DEV)
    ops.l2_argmin_tc_split(zd, cbd, pack, K, got, q, splits=S)
    ref = torch.empty(T, dtype=torch.int64, device=DEV)
    ops.l2_argmin_tc(zd, cbd, pack, K, ref)
    return got, q, ref, z, cb


@pytest.mark.parametrize('T', [1, 64, 100, 1024, 4097])
@pytest.mark.parametrize('K,E', [(2048, 256), (16384, 128), (2048, 512), (16384, 256)])
def test_split_argmin_equals_fp64_and_unsplit(T, K, E):
    for S in sorted({1, 2, 3, 7, K // 128}):
        got, q, ref, z, cb = _split_case(T, K, E, S, 'random', T + K + E + S)
        want = _argmin64(z.to(DEV), cb.to(DEV), K)
        assert torch.equal(got, ref), (S, (got != ref).sum().item())
        assert torch.equal(got, want), (S, (got != want).sum().item())
        assert torch.equal(q, cb.to(DEV)[got])


@pytest.mark.parametrize('kind', ['duplicates', 'constant', 'equal_row'])
@pytest.mark.parametrize('S', [2, 3, 7, 16])
def test_split_argmin_adversarial(kind, S):
    T, K, E = 100, 2048, 256
    got, _, ref, z, cb = _split_case(T, K, E, S, kind, S)
    want = _argmin64(z.to(DEV), cb.to(DEV), K)
    assert torch.equal(got, want) and torch.equal(got, ref)
    if kind == 'constant':
        assert (got == 0).all()


# --------------------------------------------------------------------------- the model vs the reference's outputs
def _cmp(t, g, key):
    s = golden_sample(t, g, key)
    return ((s - g[key].float()).abs().max() / g[key + '_absmax']).item(), psnr(s, g[key])


@pytest.mark.parametrize('name', FIXTURES)
def test_methods_against_reference_golden(models, name):
    from oracle.make_rqvae_golden import golden_images
    g = load_golden(name)
    m = models[g['config']]
    x = golden_images(g['seed'], g['b'], g['H'], g['W']).to(DEV)
    res = {}
    z_e = m.encode(x)
    res['z_e'] = _cmp(z_e, g, 'z_e')[0]
    out, loss, code = m(x)
    assert out.shape == (g['b'], 3, g['H'], g['W']) and code.shape == g['codes'].shape and code.dtype == torch.int64
    ref_code = g['codes'].long()
    res['code_agree'] = (code.cpu() == ref_code).float().mean().item()
    # depth 0 codes must match wherever the reference's margin exceeds what our error dz in that token's z_e can move
    # it: d_k = |z - e_k|^2 moves by 2 <dz, z - e_k> + |dz|^2, so the margin of the two nearest codes by at most
    # 4 |dz| |z - e_1| + 2 |dz|^2 (to first order in |e_1 - e_2|); deeper depths see residuals of the earlier codes and
    # are checked by agreement
    zr = g['z_e'].double().view(z_e.shape)
    dz = (z_e.double().cpu() - zr).norm(dim=-1)
    cb = m.quantizer.codebooks._modules['0'].weight.detach().double().cpu()
    reach = (zr - cb[ref_code[..., 0]]).norm(dim=-1)
    confident = g['margin'][..., 0].double() > 4 * dz * reach + 2 * dz * dz
    res['confident'] = confident.float().mean().item()
    same_conf = (code[..., 0].cpu() == ref_code[..., 0])[confident].all().item()
    res['loss'] = abs(loss.item() - g['quant_loss'].item()) / g['quant_loss'].item()
    # the reference's own codes through decode_code and the partial decodes
    for key, fn in (('out_code', lambda: m.decode_code(ref_code.to(DEV))),
                    ('out_select1', lambda: m.decode_partial_code(ref_code.to(DEV), 1, 'select')),
                    ('out_add1', lambda: m.decode_partial_code(ref_code.to(DEV), 1, 'add'))):
        res[key + '_err'], res[key + '_psnr'] = _cmp(fn(), g, key)
    if 'soft' in g:
        soft, soft_code = m.get_soft_codes(x, 1.0)
        assert soft.shape == (*code.shape, m.arch.n_embed)
        res['soft_code_agree'] = (soft_code.cpu() == g['soft_codes'].long()).float().mean().item()
        assert torch.equal(soft_code, code)
    print('%s: %s' % (name, res))
    assert res['z_e'] < (3e-2 if m.arch.num_levels > 4 else 2.5e-2) and same_conf and res['code_agree'] > 0.8 and res['loss'] < 5e-2
    for key in ('out_code', 'out_select1', 'out_add1'):
        assert res[key + '_psnr'] > 35.0 and res[key + '_err'] < 8e-2, key
    if 'soft' in g:
        assert res['soft_code_agree'] > 0.8


# --------------------------------------------------------------------------- identities
@pytest.mark.parametrize('cfg,H,W', [('r1', 256, 128), ('r2', 64, 128)])
def test_method_identities(models, cfg, H, W):
    m = models[cfg]
    eng = m.engine()
    x = torch.rand(2, 3, H, W, generator=torch.Generator().manual_seed(H + W)).to(DEV)
    out, loss, code = m(x)
    D, E = m.arch.depth, m.arch.embed_dim
    assert torch.equal(m.get_codes(x), code)
    assert torch.equal(m.decode_code(code), out)
    assert torch.equal(m.decode_partial_code(code, D - 1, 'add'), out)
    assert torch.equal(m.forward_partial_code(x, 1, 'select'), m.decode_partial_code(code, 1, 'select'))
    assert torch.equal(m.forward_partial_code(x, 0, 'add'), m.decode_partial_code(code, 0, 'select'))
    assert torch.equal(m.get_codesbt(x.view(1, 2, 3, H, W)), code)
    emb, none = m.get_code_emb_with_depth(code)
    assert none is None and emb.shape == (*code.shape, E)
    # embed_code sums the depth rows on the device in depth order, fp32: the same order on the host gives equal bits
    acc = emb[..., 0, :].clone()
    for d in range(1, D):
        acc = acc + emb[..., d, :]
    assert torch.equal(acc.view(-1, E), eng.embed_code(code))
    z_q, loss2, code2 = m(x, code_only=True)
    assert torch.equal(code2, code) and torch.equal(loss2, loss) and z_q.shape == (*code.shape[:3], E)
    assert torch.equal(m.decode(z_q), out)
    # each depth's code is the exact nearest row of its own codebook to the residual the earlier depths left
    r = m.encode(x).double().view(-1, E)
    for d in range(D):
        cb = m.quantizer.codebooks._modules[str(d)].weight.detach().double()[:-1]
        dist = (r.pow(2).sum(1, keepdim=True) - 2 * r @ cb.t() + cb.pow(2).sum(1)[None])
        best = dist.min(1).values
        got = dist.gather(1, code.view(-1, D)[:, d:d + 1]).squeeze(1)
        assert ((got - best) <= 1e-3 * (1 + best.abs())).all(), d
        r = r - cb[code.view(-1, D)[:, d]]
    for i in range(2):
        o, _, c = m(x[i:i + 1])
        assert torch.equal(c, code[i:i + 1]) and torch.equal(o, out[i:i + 1])


def test_separate_codebook_sizes_are_respected(models):
    """R2's depths have 512, 1024 and 256 codes: no code exceeds its own codebook, and a depth-2 code of its padding
    row (index 256) decodes like the reference's padding row."""
    m = models['r2']
    x = torch.rand(4, 3, 128, 128, generator=torch.Generator().manual_seed(3)).to(DEV)
    code = m.get_codes(x)
    for d, k in enumerate((512, 1024, 256)):
        assert int(code[..., d].max()) < k
    c = code.clone()
    c[..., 2] = 256
    emb, _ = m.get_code_emb_with_depth(c)
    pad = m.quantizer.codebooks._modules['2'].weight.detach()[256]
    assert torch.equal(emb[..., 2, :], pad.expand_as(emb[..., 2, :]).float())
