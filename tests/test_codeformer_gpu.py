"""VQAutoEncoder and CodeFormer on the H100: the two new kernel paths (the generator tail without SiLU and the
VectorQuantizer statistics) against fp64 evaluations, both bindings of each new entry point, and the models against the
reference's own outputs (tests/golden/vqgan_ref_*.pt, codeformer_ref_*.pt).

Bounds: the conv tail 1e-2 * max|ref| (bf16 operands, fp32 accumulation); z, lq_feat and logits 3e-2 * max|ref|, the
bound DESIGN §2 gives the other models' latents; images compared by PSNR against max|ref| as the peak, > 35 dB
teacher-forced."""
import math

import pytest
import torch

from conftest import golden_sample, load_golden

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def relerr(got, ref):
    got, ref = got.double().cpu(), ref.double().cpu()
    assert got.shape == ref.shape, (got.shape, ref.shape)
    assert torch.isfinite(got).all()
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-12)).item()


def psnr(got, ref, peak):
    mse = (got.float().cpu() - ref.float().cpu()).pow(2).mean().item()
    return 99.0 if mse == 0 else 10 * math.log10(peak * peak / mse)


@pytest.fixture(scope='module')
def vq():
    from archs import VQAutoEncoder
    return VQAutoEncoder().to(DEV).eval()


@pytest.fixture(scope='module')
def cf():
    from archs import CodeFormer
    return CodeFormer().to(DEV).eval()


# --------------------------------------------------------------------------- the generator tail without SiLU
def _tail_inputs(F, H, W, seed):
    from pgtformer_b200 import ops
    from pgtformer_b200.engine import _pack_conv
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(F, H, W, 64, generator=g) * 2 + 0.5).to(DEV).bfloat16()
    gamma, beta = 1 + 0.2 * torch.randn(64, generator=g), 0.1 * torch.randn(64, generator=g)
    w = torch.randn(3, 64, 3, 3, generator=g) / 24
    bias = 0.05 * torch.randn(3, generator=g)
    ab = ops.groupnorm_ab(x, gamma.to(DEV), beta.to(DEV), torch.empty(F * 2 * 64, device=DEV))
    return x, gamma, beta, w, bias, ab, _pack_conv(w.to(DEV))


@pytest.mark.parametrize('F,H,W', [(1, 512, 512), (2, 64, 48), (3, 16, 8)])
def test_conv_tail_without_silu_against_fp64(F, H, W):
    from pgtformer_b200 import ops
    x, gamma, beta, w, bias, ab, wp = _tail_inputs(F, H, W, F * H + W)
    out = torch.empty(F, 3, H, W, device=DEV)
    assert ops.conv_out_gn(x, ab, wp, 3, bias.to(DEV), out, silu=False) is not None
    xd = x.double().cpu().permute(0, 3, 1, 2)
    y = torch.nn.functional.group_norm(xd, 32, gamma.double(), beta.double(), eps=1e-6)
    ref = torch.nn.functional.conv2d(y, w.double(), bias.double(), padding=1)
    e = relerr(out, ref)
    ys = torch.nn.functional.silu(y)
    e_silu = relerr(out, torch.nn.functional.conv2d(ys, w.double(), bias.double(), padding=1))
    print('conv tail without SiLU F%d %dx%d: %.3e of max|ref| (against the SiLU formula: %.3e)' % (F, H, W, e, e_silu))
    assert e < 1e-2 and e_silu > 10 * e


@pytest.mark.parametrize('F,H,W', [(1, 512, 512), (2, 64, 48)])
def test_conv_tail_bindings_and_silu_bits(F, H, W):
    """pgt_conv_out_gn_act(silu = 1) is pgt_conv_out_gn bit for bit; torch.ops.pgt.conv_out_gn_act gives the ctypes bits."""
    from pgtformer_b200 import _lib, ops, torch_ops
    x, gamma, beta, w, bias, ab, wp = _tail_inputs(F, H, W, 7)
    b = bias.to(DEV)
    lib = _lib.load()
    outs = {}
    for silu in (0, 1):
        o = torch.empty(F, 3, H, W, device=DEV)
        _lib.check(lib.pgt_conv_out_gn_act(ops._p(x), F, H, W, 64, x.stride(2), ops._p(ab), ops._p(wp), wp.stride(0), 3,
                                           ops._p(b), ops._p(o), silu, ops._stream(x)))
        t = torch.empty_like(o)
        torch_ops.load().conv_out_gn_act(x, ab, wp, 3, b, bool(silu), t)
        assert torch.equal(o, t)
        outs[silu] = o
    old = torch.empty(F, 3, H, W, device=DEV)
    _lib.check(lib.pgt_conv_out_gn(ops._p(x), F, H, W, 64, x.stride(2), ops._p(ab), ops._p(wp), wp.stride(0), 3,
                                   ops._p(b), ops._p(old), ops._stream(x)))
    assert torch.equal(outs[1], old) and not torch.equal(outs[0], old)
    assert torch.equal(ops.conv_out_gn(x, ab, wp, 3, b, torch.empty_like(old)), old)


# --------------------------------------------------------------------------- VectorQuantizer statistics
def _vq_case(b, HW, K, E, seed):
    g = torch.Generator().manual_seed(seed)
    cb = torch.randn(K, E, generator=g)
    cb[7] = cb[3]                                               # duplicated rows: the first index wins
    cb[K - 1] = cb[0]
    z = torch.randn(b * HW, E, generator=g) * 0.8
    z[0] = cb[3] + 1e-3 * torch.randn(E, generator=g)
    z[5] = cb[0] + 1e-3 * torch.randn(E, generator=g)
    return z.to(DEV), cb.to(DEV)


def _vq_run(z, cb, HW, beta, usage, binding='ctypes'):
    from pgtformer_b200 import ops, torch_ops
    T, E = z.shape
    K = cb.shape[0]
    codes = torch.empty(T, dtype=torch.int64, device=DEV)
    ops.l2_argmin_tc(z, cb, ops.codebook_pack(cb, K), K, codes)
    o = dict(scalars=torch.empty(3, device=DEV), zq_nchw=torch.empty(T // HW, E, HW, device=DEV),
             zq_bf16=torch.empty(T, E, device=DEV, dtype=torch.bfloat16), min_enc=torch.empty(T, K, device=DEV),
             scores=torch.empty(T, device=DEV))
    if binding == 'ctypes':
        ops.vq_stats(z, cb, codes, HW, beta, o['scalars'], zq_nchw=o['zq_nchw'], zq_bf16=o['zq_bf16'],
                     min_enc=o['min_enc'], scores=o['scores'], usage=usage)
    else:
        torch_ops.load().vq_stats(z, cb, codes, HW, beta, o['scalars'], o['zq_nchw'], o['zq_bf16'], o['min_enc'],
                                  o['scores'], usage)
    return codes, o


@pytest.mark.parametrize('b,HW,K,E', [(1, 256, 1024, 256), (4, 1024, 1024, 256), (3, 96, 512, 128)])
def test_vq_stats_against_fp64(b, HW, K, E):
    z, cb = _vq_case(b, HW, K, E, b * HW + K)
    T = b * HW
    usage = torch.zeros(K, dtype=torch.int32, device=DEV)
    codes, o = _vq_run(z, cb, HW, 0.25, usage)
    zd, cd = z.double(), cb.double()
    d = (zd * zd).sum(1, keepdim=True) + (cd * cd).sum(1)[None] - 2 * zd @ cd.t()
    dmin, ref_codes = d.min(1)
    assert torch.equal(codes, ref_codes) and codes[0] == 3 and codes[5] == 0
    # the straight-through value: the same fp32 expression on the CPU, bit for bit
    e = cb.cpu()[codes.cpu()]
    st = z.cpu() + (e - z.cpu())
    assert torch.equal(o['zq_nchw'].cpu(), st.view(b, HW, E).permute(0, 2, 1))
    assert torch.equal(o['zq_bf16'].cpu(), st.bfloat16())
    assert torch.equal(o['min_enc'], torch.nn.functional.one_hot(codes, K).float())
    counts = torch.bincount(codes, minlength=K).int()
    assert torch.equal(usage, counts)
    torch.testing.assert_close(o['scores'].double(), torch.exp(-dmin / 10), rtol=1e-5, atol=0)
    m = ((cd[codes] - zd) ** 2).mean()
    p = counts.double() / T
    ref = torch.stack([m + 0.25 * m, torch.exp(-(p * torch.log(p + 1e-10)).sum()), d.mean()])
    print('vq stats T %d K %d E %d: %s vs fp64 %s' % (T, K, E, o['scalars'].tolist(), ref.tolist()))
    torch.testing.assert_close(o['scalars'].double(), ref, rtol=2e-6, atol=0)
    _vq_run(z, cb, HW, 0.25, usage)                            # usage accumulates over calls
    assert torch.equal(usage, 2 * counts)


def test_vq_stats_bindings_give_identical_bits():
    z, cb = _vq_case(2, 256, 1024, 256, 3)
    u1, u2 = torch.zeros(1024, dtype=torch.int32, device=DEV), torch.zeros(1024, dtype=torch.int32, device=DEV)
    c1, o1 = _vq_run(z, cb, 256, 0.25, u1)
    c2, o2 = _vq_run(z, cb, 256, 0.25, u2, binding='torch')
    assert torch.equal(c1, c2) and torch.equal(u1, u2)
    for k in o1:
        assert torch.equal(o1[k], o2[k]), k


# --------------------------------------------------------------------------- fused GroupNorm statistics at frame edges
@pytest.mark.parametrize('H,W,C,ksize', [(32, 48, 256, 3), (16, 24, 256, 3), (32, 48, 256, 2), (16, 24, 256, 2)])
def test_no_fused_statistics_where_tiles_pass_the_frame_edge(vq, H, W, C, ksize):
    """Where a conv's 128-pixel tile grid does not divide the frame (the 256-channel levels of a 256 x 384 VQGAN input:
    32 x 4 tiles over 48 columns) the epilogue would sum rows past the frame's edge into the GroupNorm statistics.
    pgt_conv_tiles_exact reports no tiles there, and the VQGAN engine then normalises from the tensor itself; where
    the grid divides the frame it keeps the fused statistics."""
    from pgtformer_b200 import ops
    assert ops.conv_tiles_per_frame(H, W, C, ksize, 1, 1) > 0
    assert ops.conv_tiles_exact(H, W, C, ksize, 1, 1) == 0
    eng = vq.engine()
    assert eng._stats_tiles(H, W, C, ksize, 1, 1) == 0
    assert eng._stats_tiles(32, 64, C, ksize, 1, 1) == ops.conv_tiles_per_frame(32, 64, C, ksize, 1, 1) > 0
    x = torch.randn(2, H, W, C, generator=torch.Generator().manual_seed(H + W)).to(DEV).bfloat16()
    p = 'encoder.blocks.13'                                     # a 256 -> 256 ResBlock
    if C == 256 and ksize == 3:
        y = eng.td_resblock(x, p, C, gn_next=True, shortcut='conv_out')
        assert getattr(y, '_pgt_gn', None) is None
        from oracle.vqgan_oracle import res_block
        sd = {k: v.double() for k, v in vq.state_dict().items() if k.startswith(p + '.')}
        ref = res_block(sd, p, x.double().permute(0, 3, 1, 2)).permute(0, 2, 3, 1)
        e = relerr(y, ref)
        print('ResBlock at %d x %d: %.3e of max|ref|' % (H, W, e))
        assert e < 1.5e-2


# --------------------------------------------------------------------------- the models against the reference
@pytest.mark.parametrize('name', ['vqgan_ref_b1_512x512_seed51.pt', 'vqgan_ref_b2_256x384_seed52.pt'])
def test_vqgan_against_reference_golden(vq, name):
    from oracle.make_codeformer_golden import golden_images
    g = load_golden(name)
    x = golden_images(g['seed'], g['b'], g['H'], g['W']).to(DEV)
    vq.quantize.reset_usage()
    out, loss, st = vq(x)
    usage = vq.quantize.usage.clone()
    z = vq.engine().last_z.permute(0, 3, 1, 2)
    quant, loss2, st2 = vq(x, code_only=True)
    assert torch.equal(loss, loss2) and torch.equal(st['min_encoding_indices'], st2['min_encoding_indices'])
    assert torch.equal(vq.quantize.usage, 2 * usage)
    codes = st['min_encoding_indices'].view(-1).cpu()
    ref_codes = g['codes'].long()
    zs = golden_sample(z, g, 'z')
    res = {'z': ((zs - g['z']).abs().max() / g['z_absmax']).item()}
    rms = (zs - g['z']).pow(2).mean().sqrt().item()
    # a code is decided with confidence when the reference's top-2 distance margin exceeds 3x the distance error our z
    # error causes (about 2 rms(dz) |z - e| for an error uncorrelated with z - e)
    emb = vq.quantize.embedding.weight.detach()
    reach = (z.permute(0, 2, 3, 1).reshape(-1, emb.shape[1]) - emb[ref_codes.to(DEV)]).norm(dim=1).cpu()
    confident = g['margin'] > 3 * 2 * rms * reach
    res.update(code_agree=(codes == ref_codes).float().mean().item(), confident=confident.float().mean().item())
    # quant = z + (e - z) is the code row where the codes agree; compare it there
    b, _, hh, ww = quant.shape
    same = (codes == ref_codes).view(b, 1, hh, ww).expand(quant.shape).contiguous().float()
    keep = golden_sample(same, g, 'quant') > 0
    res['quant'] = ((golden_sample(quant, g, 'quant') - g['quant'])[keep].abs().max() / g['quant_absmax']).item()
    res['out_psnr'] = psnr(golden_sample(out, g, 'out'), g['out'].float(), g['out_absmax'])
    # teacher-forced: the reference's codes, so the counts, the perplexity and the loss's code rows are the reference's
    usage_tf = torch.zeros(1024, dtype=torch.int32, device=DEV)
    out_tf, loss_tf, st_tf = vq.engine().forward(x, force_codes=ref_codes, usage=usage_tf)
    res['out_psnr_tf'] = psnr(golden_sample(out_tf, g, 'out'), g['out'].float(), g['out_absmax'])
    for key, v in (('loss', loss_tf), ('perplexity', st_tf['perplexity']), ('mean_distance', st_tf['mean_distance'])):
        res[key] = abs(v.item() - g[key].item()) / abs(g[key].item())
    assert torch.equal(st_tf['mean_distance'], st['mean_distance'])          # a function of z alone
    print('%s: %s' % (name, res))
    assert out.shape == (g['b'], 3, g['H'], g['W']) and out.dtype == torch.float32
    assert quant.shape == (g['b'], 256, g['H'] // 32, g['W'] // 32) and quant.dtype == torch.float32
    assert st['min_encodings'].shape == (codes.numel(), 1024) and st['min_encoding_scores'].shape == (codes.numel(), 1)
    assert res['z'] < 3e-2 and res['quant'] < 1e-6 and res['out_psnr_tf'] > 35.0
    assert (codes == ref_codes)[confident].all() and res['code_agree'] > 0.9
    assert torch.equal(usage_tf.cpu(), g['usage'].int()) and res['perplexity'] < 1e-5
    assert res['loss'] < 3e-3 and res['mean_distance'] < 1.5e-3


def _cf_logits_err(logits, g):
    rows = g['logit_rows']
    return ((logits.reshape(-1, logits.shape[-1])[rows.to(DEV)].cpu() - g['logits_sel']).abs().max()
            / g['logits_absmax']).item()


@pytest.mark.parametrize('name', ['codeformer_ref_b1_512_seed61.pt', 'codeformer_ref_b2_512_seed62.pt'])
def test_codeformer_against_reference_golden(cf, name):
    from oracle.make_codeformer_golden import golden_images
    g = load_golden(name)
    b = g['b']
    x = golden_images(g['seed'], b, 512, 512).to(DEV)
    logits, lq = cf(x, code_only=True)
    assert logits.shape == (b, 256, 1024) and lq.shape == (b, 256, 16, 16)
    res = {'lq_feat': ((golden_sample(lq, g, 'lq_feat') - g['lq_feat']).abs().max() / g['lq_feat_absmax']).item(),
           'logits': _cf_logits_err(logits, g)}
    err = (logits.reshape(-1, 1024)[g['logit_rows'].to(DEV)].cpu() - g['logits_sel']).abs().max().item()
    codes = logits.argmax(-1).reshape(-1).cpu()
    ref_codes = g['codes'].long()
    confident = g['margin'] > 3 * 2 * err
    res.update(code_agree=(codes == ref_codes).float().mean().item(), confident=confident.float().mean().item())
    for i, (w, adain) in enumerate(g['cases']):
        out, logits2, lq2 = cf(x, w=w, adain=adain)
        assert torch.equal(logits2, logits) and torch.equal(lq2, lq)
        assert torch.equal(cf.engine().last_codes.reshape(-1).cpu(), codes)
        out_tf, _, _ = cf(x, w=w, adain=adain, force_codes=ref_codes.view(b, 256))
        res['psnr_tf_w%g_adain%d' % (w, adain)] = psnr(golden_sample(out_tf, g, 'out%d' % i), g['out%d' % i].float(),
                                                        g['out%d_absmax' % i])
    print('%s: %s' % (name, res))
    assert res['lq_feat'] < 3e-2 and res['logits'] < 3e-2
    assert (codes == ref_codes)[confident].all() and res['code_agree'] > 0.9
    assert min(v for k, v in res.items() if k.startswith('psnr_tf')) > 35.0


# --------------------------------------------------------------------------- identities
def test_codeformer_batch_equals_per_image(cf):
    x = (torch.rand(2, 3, 512, 512, generator=torch.Generator().manual_seed(5)) * 2 - 1).to(DEV)
    outs = cf(x, w=0.5, adain=True)
    for i in range(2):
        for u, v in zip(outs, cf(x[i:i + 1], w=0.5, adain=True)):
            assert torch.equal(u[i:i + 1], v)


def test_vqgan_batch_equals_per_image(vq):
    x = (torch.rand(2, 3, 256, 384, generator=torch.Generator().manual_seed(6)) * 2 - 1).to(DEV)
    out, _, st = vq(x)
    for i in range(2):
        o, _, s = vq(x[i:i + 1])
        assert torch.equal(o, out[i:i + 1])
        assert torch.equal(s['min_encoding_indices'].view(-1), st['min_encoding_indices'].view(2, -1)[i])


def test_other_models_unchanged_by_codeformer_calls(network_g, cf, vq):
    from archs.pgtformer_arch import PGTFormer, TDCRQVAE3
    from archs.tdrqvae_arch import TDRQVAE
    opt = dict(network_g)
    opt.pop('type')
    pgt = PGTFormer(**opt).to(DEV).eval()
    tdc = TDCRQVAE3(**opt).to(DEV).eval()
    tdr = TDRQVAE(**dict(opt)).to(DEV).eval()
    x = torch.rand(3, 3, 64, 64, generator=torch.Generator().manual_seed(9)).to(DEV)
    a = [t.clone() for t in pgt(x, w=1, adain=True)]
    av = [t.clone() for t in tdc(x)]
    ar = [t.clone() for t in tdr(x.view(1, 3, 3, 64, 64))]
    cf(torch.rand(1, 3, 512, 512, generator=torch.Generator().manual_seed(10)).to(DEV), w=1.0, adain=True)
    vq(torch.rand(1, 3, 256, 256, generator=torch.Generator().manual_seed(11)).to(DEV))
    for u, v in zip(a, pgt(x, w=1, adain=True)):
        assert torch.equal(u, v)
    for u, v in zip(av, tdc(x)):
        assert torch.equal(u, v)
    for u, v in zip(ar, tdr(x.view(1, 3, 3, 64, 64))):
        assert torch.equal(u, v)
