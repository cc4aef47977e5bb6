"""GPU tests of the residual quantiser at depth D > 1 (rq.cu, the depth loops of engine.py, the D-aware methods of
archs/pgtformer_arch.py).

- The quantiser against an fp64 adjudicator that runs the same fp32 residual chain: every code equal at every depth,
  residuals and aggregates bit-identical (the kernels do one IEEE fp32 subtraction / addition per element, as the
  reference's sub_ / add_ do).
- rq_embed against sequential fp32 sums, bit for bit; the strided soft codes against fp64; the sampler.
- The model methods against the reference's own outputs (tests/golden/rq_*.pt, `python -m oracle.make_rq_golden`), with
  the tolerances of the depth-1 codec tests, and the identities between the methods, bit for bit."""
import types

import pytest
import torch

from conftest import golden_sample, load_golden

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def rq_engine(cbs, shared):
    """An Engine holding only a quantiser: D codebooks [K + 1, E] (for shared, the same tensor D times)."""
    from pgtformer_b200.engine import Engine
    eng = Engine.__new__(Engine)
    K, E = cbs[0].shape[0] - 1, cbs[0].shape[1]
    eng.arch = types.SimpleNamespace(code_shape=(1, 1, len(cbs)), n_embed=K, embed_dim=E, shared_codebook=shared)
    eng.dev = torch.device(DEV)
    eng.w = {'codebook': cbs[0].to(DEV).contiguous()}
    if len(cbs) > 1:
        eng.w['codebooks'] = torch.stack([c.to(DEV) for c in (cbs[:1] if shared else cbs)]).contiguous()
    return eng


def make_codebooks(D, K, E, shared, seed, dup=False):
    g = torch.Generator().manual_seed(seed)
    cbs = []
    for d in range(1 if shared else D):
        w = torch.randn(K + 1, E, generator=g) * 0.5 ** d
        if dup:
            w[1:K:3] = w[0:K - 1:3]                    # duplicated rows: ties go to the lowest index
        w[-1].zero_()
        cbs.append(w)
    return cbs * D if shared else cbs


def fp64_chain(cbs, z):
    """The reference chain with an fp64 argmin: codes [T, D], residual before each depth, aggregates after each."""
    r, agg = z.clone(), torch.zeros_like(z)
    codes, res, aggs = [], [], []
    for cb in cbs:
        cbd = cb.to(DEV)
        e = cbd[:-1].double()
        rd = r.double()
        dist = (rd * rd).sum(1, keepdim=True) + (e * e).sum(1)[None] - 2.0 * (rd @ e.t())
        c = dist.argmin(1)
        res.append(r.clone())
        q = cbd[c]
        r = r - q
        agg = agg + q
        codes.append(c)
        aggs.append(agg.clone())
    return torch.stack(codes, 1), res, aggs


@pytest.mark.parametrize('shared', [False, True])
@pytest.mark.parametrize('D', [2, 3, 4])
@pytest.mark.parametrize('K,E', [(1024, 512), (1024, 256), (1024, 96), (300, 512), (300, 96)])
def test_quantizer_matches_the_fp64_chain(K, E, D, shared):
    T = 4097
    cbs = make_codebooks(D, K, E, shared, seed=K + E + D, dup=True)
    g = torch.Generator().manual_seed(7 * D + E)
    z = (torch.randn(T, E, generator=g) + cbs[0][torch.randint(0, K, (T,), generator=g)] * 0.5).to(DEV)
    z[5:40] = cbs[0][1].to(DEV)                         # exact hits on row 1, a copy of row 0: the tie goes to 0
    eng = rq_engine(cbs, shared)
    codes, z_q, loss = eng.quantize(z)
    ref_codes, _, aggs = fp64_chain(cbs, z)
    assert codes.shape == (T, D) and codes.dtype == torch.int64
    assert torch.equal(codes, ref_codes), (codes != ref_codes).sum(0)
    assert torch.equal(z_q, aggs[-1])
    ref_loss = torch.stack([(z - a).pow(2).mean() for a in aggs]).mean()
    assert torch.equal(loss, ref_loss)


def test_ties_go_to_the_lowest_index():
    K, E, D = 1024, 512, 2
    cbs = make_codebooks(D, K, E, False, seed=3)
    cbs[0][5] = cbs[0][4]
    cbs[1][9] = cbs[1][8]
    z = (cbs[0][5] + cbs[1][8]).repeat(300, 1).to(DEV)
    codes, _, _ = rq_engine(cbs, False).quantize(z)
    assert (codes[:, 0] == 4).all() and (codes[:, 1] == 8).all()


def test_planted_codes_are_recovered():
    """codebook d scaled by 0.5^d, z = sum_d e_d[c*_d] + small noise: every level's answer is known."""
    K, E, D, T = 1024, 512, 4, 8192
    cbs = make_codebooks(D, K, E, False, seed=11)
    g = torch.Generator().manual_seed(12)
    want = torch.randint(0, K, (T, D), generator=g)
    z = sum(cbs[d][want[:, d]] for d in range(D)) + 1e-3 * torch.randn(T, E, generator=g)
    codes, z_q, _ = rq_engine(cbs, False).quantize(z.to(DEV))
    assert torch.equal(codes.cpu(), want)
    assert ((z_q.cpu() - z).abs().max() < 1e-2)


# --------------------------------------------------------------------------- rq_embed
def seq_sum(cbs, codes, d0, d1):
    s = cbs[d0].to(DEV)[codes[:, d0]]
    for d in range(d0 + 1, d1 + 1):
        s = s + cbs[d].to(DEV)[codes[:, d]]
    return s


@pytest.mark.parametrize('shared', [False, True])
@pytest.mark.parametrize('out_dtype', [torch.float32, torch.bfloat16])
def test_rq_embed_every_mode_is_a_sequential_fp32_sum(shared, out_dtype):
    from pgtformer_b200 import ops
    K, E, D, T = 1024, 512, 4, 3001
    cbs = make_codebooks(D, K, E, shared, seed=21)
    stacked = torch.stack([c for c in (cbs[:1] if shared else cbs)]).to(DEV).contiguous()
    codes = torch.randint(0, K + 1, (T, D), generator=torch.Generator().manual_seed(2)).to(DEV)
    codes[::5] = K                                           # the padding row
    dm = codes.t().contiguous()                              # depth-major [D, T]
    for d0, d1 in [(0, D - 1), (0, 0), (0, 2), (1, 1), (3, 3), (1, 3)]:
        want = seq_sum(cbs, codes, d0, d1).to(out_dtype)
        wide = torch.zeros(T, E + 64, dtype=out_dtype, device=DEV)               # row pitch > E
        got = ops.rq_embed(codes, d0, d1, stacked, wide[:, :E], ldi=D, ldd=1)
        assert torch.equal(got, want) and (wide[:, E:] == 0).all()
        got = ops.rq_embed(dm, d0, d1, stacked, torch.empty(T, E, dtype=out_dtype, device=DEV), ldi=1, ldd=T)
        assert torch.equal(got, want)


def test_bindings_agree_on_the_rq_entries():
    from pgtformer_b200 import ops, torch_ops
    tops = torch_ops.load()
    K, E, D, T = 1024, 512, 3, 2000
    cbs = make_codebooks(D, K, E, False, seed=31)
    stacked = torch.stack(cbs).to(DEV).contiguous()
    codes = torch.randint(0, K + 1, (T, D), generator=torch.Generator().manual_seed(3)).to(DEV)
    a = ops.rq_embed(codes, 0, D - 1, stacked, torch.empty(T, E, device=DEV), ldi=D, ldd=1)
    b = torch.empty(T, E, device=DEV)
    tops.rq_embed(codes, 0, D - 1, stacked, b, D, 1)
    assert torch.equal(a, b)
    z = torch.randn(T, E, device=DEV)
    cb = stacked[1]
    r1, r2, g1, g2 = (torch.empty(T, E, device=DEV) for _ in range(4))
    g1.copy_(z)
    g2.copy_(z)
    ops.rq_residual(z, r1, codes[:, 1].contiguous(), cb, g1, False)
    tops.rq_residual(z, r2, codes[:, 1].contiguous(), cb, g2, False)
    assert torch.equal(r1, r2) and torch.equal(g1, g2)
    _, norm = ops.codebook_pack(cb, K)
    p1, p2 = torch.zeros(T, 2, K, device=DEV), torch.zeros(T, 2, K, device=DEV)
    ops.soft_codes(z, cb, norm, K, 3.0, p1[:, 1])
    tops.soft_codes(z, cb, norm, K, 3.0, p2[:, 1])
    assert torch.equal(p1, p2) and (p1[:, 0] == 0).all()
    seed = torch.tensor([5, 6], dtype=torch.int64, device=DEV)
    i1, i2 = torch.empty(T, dtype=torch.int64, device=DEV), torch.empty(T, dtype=torch.int64, device=DEV)
    ops.sample_codes(p1[:, 1], seed, i1)
    tops.sample_codes(p2[:, 1], seed, i2)
    assert torch.equal(i1, i2)


# --------------------------------------------------------------------------- soft codes
@pytest.mark.parametrize('shared', [False, True])
def test_soft_codes_per_depth_against_fp64(shared):
    """Per depth, the contract of the depth-1 soft-code tests: max|p - p64| <= 4 max|p_ref32 - p64| + 1e-6, p_ref32 the
    reference's own fp32 formula on the same residual."""
    from oracle import codec_oracle as C
    K, E, D, T = 1024, 512, 3, 2048
    cbs = make_codebooks(D, K, E, shared, seed=41)
    z = torch.randn(T, E, generator=torch.Generator().manual_seed(4)).to(DEV)
    eng = rq_engine(cbs, shared)
    for temp in (1.0, 30.0):
        p, codes = eng.soft_codes(z, temp)
        assert p.shape == (T, D, K) and p.is_contiguous() and codes.shape == (T, D)
        ref_codes, res, _ = fp64_chain(cbs, z)
        assert torch.equal(codes, ref_codes)
        assert torch.equal(codes, eng.quantize(z)[0])
        for d in range(D):
            rd, e = res[d].double(), cbs[d][:-1].to(DEV).double()
            p64 = torch.softmax(-((rd * rd).sum(1, keepdim=True) + (e * e).sum(1)[None] - 2.0 * (rd @ e.t())) / temp, -1)
            err = (p[:, d].double() - p64).abs().max().item()
            pref = C.soft_codes(cbs[d], res[d].cpu(), temp)[0].reshape(T, K).to(DEV)
            ref_err = (pref.double() - p64).abs().max().item()
            print('depth %d temp %g: max|p - p64| %.3e, reference fp32 %.3e' % (d, temp, err, ref_err))
            assert err <= 4 * ref_err + 1e-6
            assert ((p[:, d].double().sum(1) - 1).abs() < 1e-5).all()


def test_sampler_is_reproducible_and_cold_samples_are_the_argmin():
    K, E, D, T = 1024, 512, 3, 2048
    cbs = make_codebooks(D, K, E, False, seed=51)
    z = torch.randn(T, E, generator=torch.Generator().manual_seed(5)).to(DEV)
    eng = rq_engine(cbs, False)
    torch.manual_seed(9)
    p1, s1 = eng.soft_codes(z, 1.0, stochastic=True)
    torch.manual_seed(9)
    p2, s2 = eng.soft_codes(z, 1.0, stochastic=True)
    _, s3 = eng.soft_codes(z, 1.0, stochastic=True)
    assert torch.equal(s1, s2) and not torch.equal(s2, s3) and torch.equal(p1, p2)
    assert s1.min() >= 0 and s1.max() < K
    _, cold = eng.soft_codes(z, 1e-4, stochastic=True)
    assert torch.equal(cold, eng.quantize(z)[0])


# --------------------------------------------------------------------------- against the reference
def test_rq_bottleneck_alone_matches_the_reference():
    """The reference RQBottleneck on seeded z, T = 4096, K = 1024, E = 512, D = 4 (separate codebooks)."""
    from oracle.make_rq_golden import rq_inputs
    g = load_golden('rq_bottleneck_T4096_K1024_E512_D4_seed41.pt')
    z, cbs = rq_inputs(g['T'], g['K'], g['E'], g['D'], g['seed'])
    eng = rq_engine(cbs, False)
    z = z.to(DEV)
    codes, z_q, _ = eng.quantize(z)
    ref = g['codes']
    agree = (codes.cpu() == ref).all(1)
    print('RQBottleneck alone: tokens with all %d codes equal %.4f' % (g['D'], agree.float().mean().item()))
    assert agree.float().mean() > 0.99
    # teacher-forced: the fp32 chain of the reference's codes is what the kernels compute for those codes
    _, _, aggs = fp64_chain(cbs, z)
    for d in range(g['D']):
        s = golden_sample(aggs[d], g, 'quant_%d' % d)
        keep = agree.repeat_interleave(g['E'])[::g['quant_%d_stride' % d]]
        assert torch.equal(s[keep], g['quant_%d' % d][keep])
    assert torch.equal(z_q, aggs[-1])


CODEC = {'d2_separate': ('rq_tdcrqvae3_d2_separate_b1_64_seed53.pt', 'rq_tdcrqvae3_d2_separate_b2_128_seed63.pt', 2, False),
         'd4_shared': ('rq_tdcrqvae3_d4_shared_b1_64_seed55.pt', 'rq_tdcrqvae3_d4_shared_b2_128_seed65.pt', 4, True)}


def _net(network_g, depth, shared):
    g = dict(network_g)
    g.pop('type', None)
    g['code_shape'] = [32, 32, depth]
    g['shared_codebook'] = shared
    return g


@pytest.fixture(scope='module', params=list(CODEC))
def codec(request, network_g):
    from archs.pgtformer_arch import PGTFormer
    small, big, D, shared = CODEC[request.param]
    m = PGTFormer(**_net(network_g, D, shared)).to(DEV)
    m.eval()
    return m, load_golden(small), load_golden(big), D


def relerr(got, ref):
    got, ref = got.float().cpu(), ref.float().cpu()
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-12)).item()


def psnr(got, ref):
    mse = (got.float().cpu() - ref.float().cpu()).pow(2).mean().item()
    return 99.0 if mse == 0 else 10 * torch.log10(torch.tensor(1.0 / mse)).item()


def test_codec_methods_match_the_reference(codec):
    from oracle.make_golden import golden_input
    from oracle.make_rq_golden import code_map
    m, g, _, D = codec
    x = golden_input(g['seed'], 1, g['H']).to(DEV)
    z_e = m.encode(x)
    assert relerr(z_e, g['z_e']) < 2.5e-2
    # teacher-forced quantiser on the reference's own z_e: codes equal where the fp32 chain is decided, z_q bit-equal
    eng = m.engine()
    codes, z_q, loss = eng.quantize(g['z_e'].to(DEV).reshape(-1, 512))
    ref_codes = g['codes'].reshape(-1, D)
    agree = (codes.cpu() == ref_codes).all(1)
    print('%d-deep teacher-forced code agreement %.4f' % (D, agree.float().mean().item()))
    assert agree.float().mean() >= 0.95
    # the reference returns the straight-through x + (quant - x) (`archs/tdcrqvae3_arch.py:335-336`), in fp32
    ze = g['z_e'].reshape(-1, 512)
    assert torch.equal((ze + (z_q.cpu() - ze))[agree], g['z_q'].reshape(-1, 512)[agree])
    assert abs(loss.item() - g['loss'].item()) <= 1e-5 * g['loss'].item() + 1e-7 or not agree.all()
    # decoders on the reference's codes
    code = g['code']
    assert torch.equal(code, code_map(g['seed'], 3, 4, 4, D, 1024))
    out_code = m.decode_code(code.to(DEV))
    assert psnr(golden_sample(out_code, g, 'out_code'), g['out_code']) > 35.0
    assert relerr(golden_sample(out_code, g, 'out_code'), g['out_code']) < 8e-2
    out = m.decode_code(g['codes'].to(DEV))
    assert psnr(golden_sample(out, g, 'out'), g['out']) > 35.0 and relerr(golden_sample(out, g, 'out'), g['out']) < 8e-2
    for j in range(D):
        for t in ('select', 'add'):
            o = golden_sample(m.decode_partial_code(code.to(DEV), j, t), g, 'partial_%s_%d' % (t, j))
            ref = g['partial_%s_%d' % (t, j)]
            assert psnr(o, ref) > 35.0 and relerr(o, ref) < 8e-2, (j, t)
    emb, none = m.get_code_emb_with_depth(code.to(DEV))
    assert none is None and emb.shape == (3, 4, 4, D, 512)
    assert torch.equal(golden_sample(emb, g, 'emb_with_depth'), g['emb_with_depth'])
    # soft codes, teacher-forced on the reference's z_e: where the codes agree the residual chains are the same, so the
    # probabilities differ only by the two fp32 distance computations
    for i, temp in enumerate(g['temps']):
        p, c = eng.soft_codes(g['z_e'].to(DEV).reshape(-1, 512), temp)
        same = (c.cpu() == g['soft_code_codes'][i].reshape(-1, D)).all(-1)
        assert same.float().mean() >= 0.95
        ps, refs = golden_sample(p.view(3, 4, 4, D, 1024), g, 'soft_code_%d' % i), g['soft_code_%d' % i]
        keep = same.repeat_interleave(D * 1024)[::g['soft_code_%d_stride' % i]]
        err = (ps[keep] - refs[keep]).abs().max().item()
        print('soft codes temp %g: %.4f tokens with equal codes, max|p - p_ref| %.3e' % (temp, same.float().mean(), err))
        assert err < 1e-3
        p, c = m.get_soft_codes(x.view(1, 3, 3, 64, 64), temp=temp)
        assert p.shape == (3, 4, 4, D, 1024) and torch.equal(c, m.get_codes(x))


def test_codec_128_two_clips(codec):
    from oracle.make_golden import golden_input
    m, _, g, D = codec
    x = golden_input(g['seed'], g['b'], g['H']).to(DEV)
    z_q, loss, codes = m.forward_vq(x, code_only=True)
    assert codes.shape == (6, 8, 8, D)
    agree = (codes.cpu() == g['codes']).all(-1).float().mean().item()
    print('128^2 b=2 depth %d: all-depth code agreement %.4f' % (D, agree))
    assert (codes[..., 0].cpu() == g['codes'][..., 0]).float().mean() >= 0.85
    out = m.decode_code(g['codes'].to(DEV))
    s = golden_sample(out, g, 'out')
    assert psnr(s, g['out']) > 35.0 and ((s - g['out']).abs().max() / g['out_absmax']).item() < 8e-2


def test_codec_identities(codec):
    from oracle.make_golden import golden_input
    m, g, _, D = codec
    x = golden_input(7, 2, 64).to(DEV)
    out, loss, codes = m.forward_vq(x)
    assert codes.shape == (6, 4, 4, D) and codes.dtype == torch.int64
    assert torch.equal(m.get_codes(x), codes)
    assert torch.equal(m.decode_partial_code(codes, D - 1, 'add'), m.decode_code(codes))
    assert torch.equal(m.forward_partial_code(x, D - 1, 'add'), m.decode_code(codes))
    assert torch.equal(m.forward_partial_code(x, 0, 'select'), m.decode_partial_code(codes, 0, 'select'))
    one = [m.forward_vq(x[3 * i:3 * i + 3]) for i in range(2)]
    assert torch.equal(torch.cat([o[0] for o in one]), out) and torch.equal(torch.cat([o[2] for o in one]), codes)
    emb, _ = m.get_code_emb_with_depth(codes)
    s = emb[..., 0, :]
    for d in range(1, D):
        s = s + emb[..., d, :]
    assert torch.equal(s.reshape(-1, 512), m.engine().embed_code(codes))
    with pytest.raises(AssertionError):
        m.decode_partial_code(codes, D)


# --------------------------------------------------------------------------- PGTFormer at depth 2
@pytest.fixture(scope='module')
def pgt2(network_g):
    from archs.pgtformer_arch import PGTFormer
    m = PGTFormer(**_net(network_g, 2, True)).to(DEV)
    m.eval()
    return m


@pytest.mark.parametrize('name', ['rq_pgtformer_d2_b1_64_seed71.pt', 'rq_pgtformer_d2_b2_128_seed72.pt'])
def test_pgtformer_depth2_teacher_forced(pgt2, name):
    from oracle.make_golden import golden_input
    g = load_golden(name)
    x = golden_input(g['seed'], g['b'], g['H']).to(DEV)
    out, logits, lq = pgt2(x, w=1.0, adain=True)
    Fr, h = 3 * g['b'], g['H'] // 16
    assert logits.shape == (Fr, h, h, 2, 1024) and lq.shape == (Fr, h, h, 512)
    codes = pgt2.engine().last_codes
    assert torch.equal(codes, logits.argmax(-1))
    agree = (codes.cpu() == g['codes']).float().mean().item()
    print('PGTFormer depth 2 %s: code agreement %.4f' % (name, agree))
    assert agree > 0.85
    assert relerr(golden_sample(lq, g, 'lq_feat'), g['lq_feat']) < 2.5e-2
    assert relerr(golden_sample(logits, g, 'logits'), g['logits']) < 2.5e-2
    out_tf, _, _ = pgt2(x, w=1.0, adain=True, force_codes=g['codes'].to(DEV))
    s = golden_sample(out_tf, g, 'out')
    print('teacher-forced PSNR %.1f dB' % psnr(s, g['out']))
    assert psnr(s, g['out']) > 35.0 and relerr(s, g['out']) < 8e-2
    # graphed replay gives the eager bits
    pgt2.cuda_graph = True
    try:
        assert torch.equal(pgt2(x, w=1.0, adain=True)[0], out)
    finally:
        pgt2.cuda_graph = False


def test_pgtformer_code_only_and_code_sum(pgt2):
    from oracle.make_golden import golden_input
    x = golden_input(3, 1, 64).to(DEV)
    logits, lq = pgt2(x, code_only=True)
    assert logits.shape == (3, 4, 4, 2, 1024)
    out, logits2, _ = pgt2(x)
    assert torch.equal(logits, logits2)
    codes = logits.argmax(-1)
    out_f, _, _ = pgt2(x, force_codes=codes)
    assert torch.equal(out_f, out)


# --------------------------------------------------------------------------- depth 1 is untouched
def test_depth1_models_unchanged_after_deep_models(network_g, codec, pgt2):
    from archs.pgtformer_arch import PGTFormer
    from oracle.make_golden import golden_input
    opt = dict(network_g)
    opt.pop('type')
    x = golden_input(8, 1, 64).to(DEV)
    m1 = PGTFormer(**opt).to(DEV)
    m1.eval()
    before = [t.clone() for t in m1(x)] + [t.clone() for t in m1.forward_vq(x)]
    codec[0].forward_vq(x)
    codec[0](x)
    pgt2(x)
    m2 = PGTFormer(**opt).to(DEV)
    m2.eval()
    for m in (m1, m2):
        after = list(m(x)) + list(m.forward_vq(x))
        assert all(torch.equal(a, b) for a, b in zip(before, after))
    assert m1.engine().last_codes.shape == (3, 4, 4, 1) and 'codebooks' not in m1.engine().w
