"""GPU tests of the stage-I codec methods: the soft-code kernel (soft_codes.cu) against an fp64 softmax, the sampler
(codebook.cu sample_codes_kernel), the model methods against the reference's own outputs (tests/golden/
tdcrqvae3_codec_*.pt) and their isolation from PGTFormer.forward.

Soft-code accuracy: max|p - p64| <= 4 max|p_ref32 - p64| + 1e-6, where p_ref32 is the reference's own fp32 formula
(addmm distances + softmax, oracle.codec_oracle.soft_codes) on the same inputs on the CPU: the kernel must be as good as
what it replaces, within a small factor.  Model-level tolerances are those of test_model_gpu.py."""
import pytest
import torch

from conftest import golden_sample, load_golden

pytestmark = pytest.mark.gpu
DEV = 'cuda'


@pytest.fixture(scope='module')
def model(network_g):
    from archs.pgtformer_arch import PGTFormer
    opt = dict(network_g)
    opt.pop('type')
    m = PGTFormer(**opt).to(DEV)
    m.eval()
    return m


@pytest.fixture(scope='module')
def codebook(model):
    return model.quantizer.codebooks._modules['0'].weight.detach().float().cpu()          # [1025, 512], padding row last


def relerr(got, ref):
    got, ref = got.float().cpu(), ref.float().cpu()
    assert got.shape == ref.shape, (got.shape, ref.shape)
    assert torch.isfinite(got).all()
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-12)).item()


def psnr(got, ref):
    mse = (got.float().cpu() - ref.float().cpu()).pow(2).mean().item()
    return 99.0 if mse == 0 else 10 * torch.log10(torch.tensor(1.0 / mse)).item()


def kernel_soft_codes(z, cb, temp):
    from pgtformer_b200 import ops
    K = cb.shape[0] - 1
    cbd = cb.to(DEV).contiguous()
    _, norm = ops.codebook_pack(cbd, K)
    p = torch.empty(z.shape[0], K, dtype=torch.float32, device=DEV)
    return ops.soft_codes(z.to(DEV).contiguous(), cbd, norm, K, temp, p)


def check_soft_codes(z, cb, temp):
    """The accuracy, normalisation and sign contract of one soft_codes call; returns the kernel's p (CPU)."""
    from oracle import codec_oracle as C
    p = kernel_soft_codes(z, cb, temp).cpu()
    assert torch.isfinite(p).all()
    K = cb.shape[0] - 1
    zd, ed = z.to(DEV).double(), cb[:K].to(DEV).double()
    d64 = (zd * zd).sum(1, keepdim=True) + (ed * ed).sum(1)[None] - 2.0 * (zd @ ed.t())
    p64 = torch.softmax(-d64 / temp, dim=-1).cpu()
    pref = C.soft_codes(cb, z, temp)[0].reshape(p.shape)
    err, ref_err = (p.double() - p64).abs().max().item(), (pref.double() - p64).abs().max().item()
    print('soft_codes T=%d temp=%g: max|p - p64| %.3e, reference fp32 %.3e' % (z.shape[0], temp, err, ref_err))
    assert err <= 4 * ref_err + 1e-6
    assert ((p.double().sum(1) - 1.0).abs() <= 1e-5).all()
    assert (p >= 0).all()
    return p


# --------------------------------------------------------------------------- soft-code kernel vs fp64
@pytest.mark.parametrize('temp', [1.0, 10.0, 100.0, 1e-3])
def test_soft_codes_fixture_rows(codebook, temp):
    z = load_golden('tdcrqvae3_codec_b1_64_seed21.pt')['z_e'].reshape(-1, 512)
    check_soft_codes(z, codebook, temp)


def test_soft_codes_random_rows_full_size(codebook):
    """T = 49152 tokens: 16 clips of 512^2."""
    z = torch.randn(49152, 512, generator=torch.Generator().manual_seed(5)) * 0.2
    check_soft_codes(z, codebook, 1.0)


def test_soft_codes_one_hot_rows_have_exact_zeros(codebook):
    g = torch.Generator().manual_seed(6)
    code = torch.randint(0, 1024, (4096,), generator=g)
    z = codebook[code] + 1e-3 * torch.randn(4096, 512, generator=g)
    p = check_soft_codes(z, codebook, 1.0)
    assert torch.equal(p.argmax(1), code)
    assert ((p == 0).sum(1) == 1023).all() and (p.max(1).values == 1.0).all()


def test_soft_codes_duplicated_codes_get_equal_probabilities(codebook):
    cb = codebook.clone()
    cb[1:1024:2] = cb[0:1024:2]
    z = torch.randn(1024, 512, generator=torch.Generator().manual_seed(7)) * 0.5 + cb[:1024][torch.arange(1024).flip(0)] * 0.5
    p = check_soft_codes(z, cb, 10.0)
    a, b = p[:, 0::2], p[:, 1::2]
    assert ((a - b).abs() <= torch.finfo(torch.float32).eps * torch.maximum(a, b)).all()


def test_soft_codes_zero_codebook_is_uniform():
    cb = torch.zeros(1025, 512)
    z = torch.randn(300, 512, generator=torch.Generator().manual_seed(8))
    p = check_soft_codes(z, cb, 1.0)
    assert (p == 1.0 / 1024).all()


def test_soft_codes_rejects_bad_temperature_in_the_abi(codebook):
    with pytest.raises(RuntimeError, match='invalid'):
        kernel_soft_codes(torch.zeros(128, 512), codebook, float('nan'))
    with pytest.raises(RuntimeError, match='invalid'):
        kernel_soft_codes(torch.zeros(128, 512), codebook, 0.0)


# --------------------------------------------------------------------------- sampler
def _sample(p, seed):
    from pgtformer_b200 import ops
    idx = torch.empty(p.shape[0], dtype=torch.int64, device=DEV)
    return ops.sample_codes(p, torch.tensor(seed, dtype=torch.int64, device=DEV), idx)


def test_sampler_chi_square(codebook):
    """2^17 draws from one temp-10 row of the fixture against its probabilities (bins below 5 expected merged)."""
    from scipy import stats
    z = load_golden('tdcrqvae3_codec_b1_64_seed21.pt')['z_e'].reshape(-1, 512)[:1]
    row = kernel_soft_codes(z, codebook, 10.0)
    n = 1 << 17
    codes = _sample(row.expand(n, -1).contiguous(), [1234, 5678]).cpu()
    assert codes.min() >= 0 and codes.max() < 1024
    obs = torch.bincount(codes, minlength=1024).double()
    exp = row[0].double().cpu()
    exp = exp / exp.sum() * n
    big = exp >= 5
    o = torch.cat([obs[big], obs[~big].sum().view(1)])
    e = torch.cat([exp[big], exp[~big].sum().view(1)])
    if e[-1] < 5:
        o, e = torch.cat([o[:-2], o[-2:].sum().view(1)]), torch.cat([e[:-2], e[-2:].sum().view(1)])
    res = stats.chisquare(o.numpy(), e.numpy())
    print('sampler chi-square: %d bins, p-value %.4f' % (len(o), res.pvalue))
    assert big.sum() > 20 and res.pvalue > 1e-3


def test_sampler_seeds(codebook):
    z = load_golden('tdcrqvae3_codec_b1_64_seed21.pt')['z_e'].reshape(-1, 512)
    p = kernel_soft_codes(z, codebook, 100.0)
    a, b, c = _sample(p, [1, 2]), _sample(p, [1, 2]), _sample(p, [3, 2])
    assert torch.equal(a, b) and not torch.equal(a, c)


def test_sampler_never_draws_zero_probability_codes():
    g = torch.Generator().manual_seed(9)
    p = torch.rand(1 << 16, 1024, generator=g)
    p[torch.rand(1 << 16, 1024, generator=g) < 0.9] = 0.0
    p[:, -40:] = 0.0                                        # trailing zeros: the clamp must not land on them
    p[:8] = 0.0
    p[:8, 5] = 1e-30                                        # a single tiny positive entry
    pd = p.to(DEV)
    codes = _sample(pd, [11, 12])
    assert (pd.gather(1, codes[:, None]) > 0).all()
    assert (codes[:8] == 5).all()


def test_sampler_one_hot_rows():
    hot = torch.randint(0, 1024, (4096,), generator=torch.Generator().manual_seed(10)).to(DEV)
    p = torch.zeros(4096, 1024, device=DEV)
    p[torch.arange(4096, device=DEV), hot] = 1.0
    assert torch.equal(_sample(p, [5, 6]), hot)


# --------------------------------------------------------------------------- model methods vs the reference's outputs
def test_encode_decode_against_reference_golden_64(model):
    from oracle.make_golden import golden_input
    g = load_golden('tdcrqvae3_codec_b1_64_seed21.pt')
    x = golden_input(g['seed'], g['b'], g['H'])
    z_e = model.encode(x.view(1, 3, 3, 64, 64).to(DEV))
    assert z_e.dtype == torch.float32 and relerr(z_e, g['z_e']) < 2.5e-2
    assert torch.equal(z_e, model.encode(x.to(DEV)))                       # both input forms
    out = model.decode(g['z_q'].to(DEV))
    assert out.shape == g['out'].shape and out.dtype == torch.float32
    assert psnr(out, g['out']) > 35.0 and relerr(out, g['out']) < 8e-2
    out_code = model.decode_code(g['code'].to(DEV))
    assert psnr(out_code, g['out_code']) > 35.0 and relerr(out_code, g['out_code']) < 8e-2
    assert torch.equal(model.decode_partial_code(g['code'].to(DEV), 0), out_code)
    assert torch.equal(model.decode_partial_code(g['code'], 0, decode_type='add'), out_code)
    emb, none = model.get_code_emb_with_depth(g['code'])
    cb = model.quantizer.codebooks._modules['0'].weight.detach()
    assert none is None and emb.shape == (3, 4, 4, 1, 512) and torch.equal(emb, cb[g['code'].to(DEV)])


def test_encode_decode_against_reference_golden_128_b2(model):
    from oracle.make_golden import golden_input
    g = load_golden('tdcrqvae3_codec_b2_128_seed22.pt')
    x = golden_input(g['seed'], g['b'], g['H']).to(DEV)
    z_e = model.encode(x)
    s = golden_sample(z_e, g, 'z_e')
    assert ((s - g['z_e']).abs().max() / g['z_e_absmax']).item() < 2.5e-2
    out = model.decode_code(g['codes'].to(DEV))
    s = golden_sample(out, g, 'out')
    assert psnr(s, g['out']) > 35.0 and ((s - g['out']).abs().max() / g['out_absmax']).item() < 8e-2


def test_get_soft_codes_is_the_kernel_on_encode(model):
    from pgtformer_b200 import ops
    x = torch.rand(6, 3, 64, 64, generator=torch.Generator().manual_seed(13)).to(DEV)
    eng = model.engine()
    cb = eng.w['codebook']
    for t in (1.0, 10.0, 100.0):
        p, code = model.get_soft_codes(x, t)
        assert p.shape == (6, 4, 4, 1, 1024) and code.shape == (6, 4, 4, 1) and code.dtype == torch.int64
        z = model.encode(x).reshape(-1, 512)
        ref = torch.empty(z.shape[0], 1024, device=DEV)
        ops.soft_codes(z, cb, ops.codebook_pack(cb, 1024)[1], 1024, t, ref)
        assert torch.equal(p.view(-1, 1024), ref)
        assert torch.equal(code, model.get_codes(x))
    torch.manual_seed(3)
    _, s1 = model.get_soft_codes(x.view(2, 3, 3, 64, 64), 10.0, stochastic=True)
    torch.manual_seed(3)
    _, s2 = model.get_soft_codes(x, 10.0, stochastic=True)
    _, s3 = model.get_soft_codes(x, 10.0, stochastic=True)
    assert torch.equal(s1, s2) and not torch.equal(s2, s3)
    assert s1.min() >= 0 and s1.max() < 1024


def test_forward_partial_code(model):
    x = torch.rand(3, 3, 64, 64, generator=torch.Generator().manual_seed(14)).to(DEV)
    ref = model.decode_code(model.get_codes(x))
    assert torch.equal(model.forward_partial_code(x, 0), ref)
    assert torch.equal(model.forward_partial_code(x.view(1, 3, 3, 64, 64), 0, 'add'), ref)
    assert torch.equal(model.forward_vq(x)[0], ref)                        # decode(z_q) of the L2-argmin codes


# --------------------------------------------------------------------------- isolation from PGTFormer.forward
def test_encode_equals_forward_lq_feat(model):
    x = torch.rand(6, 3, 128, 128, generator=torch.Generator().manual_seed(15)).to(DEV)
    assert torch.equal(model.encode(x), model(x, code_only=True)[1])


def test_codec_calls_leave_forward_unchanged(model):
    x = torch.rand(3, 3, 64, 64, generator=torch.Generator().manual_seed(16)).to(DEV)
    a = [t.clone() for t in model(x, w=1, adain=True)]
    code = torch.randint(0, 1025, (3, 4, 4, 1), generator=torch.Generator().manual_seed(17))
    model.decode_code(code)
    model.get_soft_codes(x, 1.0, stochastic=True)
    b = model(x, w=1, adain=True)
    for u, v in zip(a, b):
        assert torch.equal(u, v)


# --------------------------------------------------------------------------- bindings
def test_torch_ops_binding_equals_ctypes_binding(codebook):
    from pgtformer_b200 import ops, torch_ops
    torch_ops.load()
    z = load_golden('tdcrqvae3_codec_b1_64_seed21.pt')['z_e'].reshape(-1, 512).to(DEV)
    cbd = codebook.to(DEV)
    norm = ops.codebook_pack(cbd, 1024)[1]
    a = torch.empty(z.shape[0], 1024, device=DEV)
    b = torch.empty_like(a)
    ops.soft_codes(z, cbd, norm, 1024, 10.0, a)
    torch.ops.pgt.soft_codes(z, cbd, norm, 1024, 10.0, b)
    assert torch.equal(a, b)
    seed = torch.tensor([7, 8], dtype=torch.int64, device=DEV)
    ia, ib = torch.empty(z.shape[0], dtype=torch.int64, device=DEV), torch.empty(z.shape[0], dtype=torch.int64, device=DEV)
    ops.sample_codes(a, seed, ia)
    torch.ops.pgt.sample_codes(a, seed, ib)
    assert torch.equal(ia, ib)
