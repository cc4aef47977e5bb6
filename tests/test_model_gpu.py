"""GPU parity of the engine's blocks and of the whole drop-in forward against the CPU oracle and
the committed golden vectors (outputs OF THE REFERENCE, tests/golden/).

Tolerances.  Kernels compute with bf16 operands / fp32 accumulation and store activations as
bf16, so a block is compared with the fp32 oracle fed the SAME bf16-rounded input and GEMM
weights; the bound is `rel * max|ref|` with rel stated per test (1 bf16 ulp is 3.9e-3 of a
value, and a block chains 6-40 kernels).  End to end the reference's own bf16-autocast forward
is 1.7e-2 off its fp64 forward on lq_feat and flips ~0.4 % of the codes at random init (SURVEY
F9); the full-forward checks therefore (a) bound lq_feat / logits, (b) report code agreement,
(c) teacher-force the golden codes to compare the decoder output.
"""
import pytest
import torch

from conftest import golden_sample, load_golden

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def relerr(got, ref):
    got, ref = got.float().cpu(), ref.float().cpu()
    assert got.shape == ref.shape, (got.shape, ref.shape)
    assert torch.isfinite(got).all()
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-12)).item()


def sampled_relerr(got, g, key):
    """relerr against a golden tensor kept as a strided sample: max |got - ref| over the sample / max |ref| overall."""
    s = golden_sample(got, g, key)
    assert torch.isfinite(got).all()
    return ((s - g[key].float()).abs().max() / max(g[key + '_absmax'], 1e-12)).item()


def psnr(got, ref):
    mse = (got.float().cpu() - ref.float().cpu()).pow(2).mean().item()
    return 99.0 if mse == 0 else 10 * torch.log10(torch.tensor(1.0 / mse)).item()


@pytest.fixture(scope='module')
def bf_sd(synth_sd):
    """Oracle weights with the GEMM / conv weights rounded to bf16 (what the kernels consume)."""
    out = {}
    for k, v in synth_sd.items():
        gemm = (k.endswith('.weight') and v.dim() in (2, 4) and 'codebooks' not in k
                and k != 'encoder.conv_in.weight' and not k.startswith('conditionnet.')) or k.endswith('in_proj_weight')
        out[k] = v.bfloat16().float() if gemm else v
    return out


@pytest.fixture(scope='module')
def model(network_g):
    from archs.pgtformer_arch import PGTFormer
    opt = dict(network_g)
    opt.pop('type')
    m = PGTFormer(**opt).to(DEV)
    m.eval()
    return m


@pytest.fixture(scope='module')
def eng(model):
    return model.engine()


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def rand_fm(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).bfloat16()


def test_state_dict_is_reference_compatible(model, synth_sd):
    sd = model.state_dict()
    assert set(sd) == set(synth_sd)
    assert all(torch.equal(sd[k].cpu(), synth_sd[k]) for k in sd)
    model.load_state_dict(synth_sd, strict=True)


@pytest.mark.parametrize('prefix,cin,cout,hw', [
    ('encoder.down.0.block.0', 64, 64, 32), ('encoder.down.1.block.0', 64, 128, 16),
    ('decoder.up.3.block.0', 512, 256, 8), ('decoder.up.0.block.0', 128, 64, 32)])
def test_td_resblock(eng, bf_sd, prefix, cin, cout, hw):
    from oracle import pgt_oracle as O
    x = rand_fm((3, hw, hw, cin), 1)
    got = eng.td_resblock(x.to(DEV), prefix, cout)
    ref = nhwc(O.td_resblock(bf_sd, prefix, x.float().permute(0, 3, 1, 2)))
    assert relerr(got, ref) < 1.5e-2


@pytest.mark.parametrize('prefix,C,hw,clips', [
    ('encoder.down.2.attn.0', 256, 16, 1), ('encoder.down.4.attn.0', 512, 8, 2), ('decoder.up.3.attn.1', 256, 16, 1),
    ('decoder.mid.attn_1', 512, 4, 1)])
def test_encoder_layer(eng, bf_sd, prefix, C, hw, clips):
    from oracle import pgt_oracle as O
    x = rand_fm((3 * clips, hw, hw, C), 2)
    got = eng.encoder_layer(x.to(DEV), prefix, 8, 2)
    ref = nhwc(O.encoder_layer(bf_sd, prefix, x.float().permute(0, 3, 1, 2), 8, 2))
    assert relerr(got, ref) < 1.5e-2


@pytest.mark.parametrize('key,C,hw', [('32', 512, 8), ('256', 128, 16)])
def test_fuse_sft(eng, bf_sd, key, C, hw):
    from oracle import pgt_oracle as O
    enc, dec = rand_fm((6, hw, hw, C), 3), rand_fm((6, hw, hw, C), 4)
    got = eng.fuse_sft(enc.to(DEV), dec.to(DEV), key, 0.8)
    ref = nhwc(O.fuse_sft(bf_sd, 'fuse_convs_dict.' + key, enc.float().permute(0, 3, 1, 2), dec.float().permute(0, 3, 1, 2), 0.8))
    assert relerr(got, ref) < 2e-2


def test_parsing_net_and_pos(eng, bf_sd):
    from oracle import pgt_oracle as O
    x = torch.rand(3, 3, 128, 128, generator=torch.Generator().manual_seed(5))
    got = eng.parse_pos(x.to(DEV))
    mean = torch.tensor(O.IMAGENET_MEAN).view(1, 3, 1, 1)
    std = torch.tensor(O.IMAGENET_STD).view(1, 3, 1, 1)
    ref = nhwc(O.conv(bf_sd, 'convpos', O.bisenet(bf_sd, 'conditionnet', (x - mean) / std)))
    assert relerr(got.view(ref.shape), ref) < 3e-2      # ~25 chained bf16 kernels with folded BatchNorm


def test_global_transformer(eng, bf_sd, arch_spec):
    from oracle import pgt_oracle as O
    arch, _ = arch_spec
    clips, hw = 2, 8
    T = clips * 3 * hw * hw
    lq, pos = rand_fm((T, 512), 6, 0.5), rand_fm((T, 512), 7, 0.5)
    got = eng.global_transformer(lq.to(DEV), pos.to(DEV), clips)
    L = 3 * hw * hw
    q = O.linear(bf_sd, 'feat_emb', lq.float()).view(clips, L, 512).transpose(0, 1)
    pp = pos.float().view(clips, L, 512).transpose(0, 1)
    for i in range(arch.n_layers):
        q = O.transformer_sa_layer(bf_sd, 'ft_layers.%d' % i, q, pp, arch.n_head)
    ref = torch.nn.functional.linear(O.layer_norm(bf_sd, 'idx_pred_layer.0', q), bf_sd['idx_pred_layer.1.weight'])
    ref = ref.transpose(0, 1).reshape(T, -1)
    assert relerr(got, ref) < 1.5e-2


def test_encoder_decoder_stages(eng, bf_sd, arch_spec):
    """At 128 x 128 and at 64 x 192, where the tile grids of several levels do not divide the frame (level 0's
    Downsample: 64-column tiles over 96 columns)."""
    from oracle import pgt_oracle as O
    arch, _ = arch_spec
    for H, W in ((128, 128), (64, 192)):
        x = torch.rand(3, 3, H, W, generator=torch.Generator().manual_seed(8))
        h, feats = eng.encoder(x.to(DEV))
        rh, rfeats = O.encoder_forward(bf_sd, arch, x)
        assert relerr(h, nhwc(rh)) < 3e-2, (H, W)
        for a, b in zip(feats, rfeats):
            assert relerr(a, nhwc(b)) < 3e-2, (H, W, tuple(a.shape))
        z = rand_fm((3, H // 16, W // 16, 256), 9, 0.5)
        efeats = [nhwc(f).bfloat16() for f in rfeats]
        out = eng.decoder(z.to(DEV), [f.to(DEV) for f in efeats], 1.0)
        ref = O.decoder_forward(bf_sd, arch, z.float().permute(0, 3, 1, 2),
                                [f.float().permute(0, 3, 1, 2) for f in efeats], 1.0)
        assert relerr(out, ref) < 4e-2 and psnr(out, ref) > 38.0, (H, W)


@pytest.mark.parametrize('fixture', ['pgtformer_ref_b1_128_seed1.pt', 'pgtformer_ref_b2_128_seed2.pt'])
def test_forward_against_reference_golden(model, fixture):
    from oracle.make_golden import golden_input
    g = load_golden(fixture)
    x = golden_input(g['seed'], g['b'], g['H']).to(DEV)
    out, logits, lq = model(x, w=1, adain=True)
    assert out.dtype == logits.dtype == lq.dtype == torch.float32
    # the fixture keeps a strided sample of each reference tensor (golden_sample checks the full shape) and max|ref|
    assert sampled_relerr(lq, g, 'lq_feat') < 2.5e-2
    assert sampled_relerr(logits, g, 'logits') < 2.5e-2
    gcodes = g['codes']
    agree = (logits.argmax(-1).cpu() == gcodes).float().mean().item()
    print('code agreement vs reference: %.4f' % agree)
    assert agree > 0.90
    # teacher-forced reference codes -> decoder output comparable with the reference's `out`
    out_tf, _, _ = model(x, w=1, adain=True, force_codes=gcodes)
    p = psnr(golden_sample(out_tf, g, 'out'), g['out'])
    print('teacher-forced PSNR vs reference out: %.2f dB' % p)
    assert p > 35.0 and sampled_relerr(out_tf, g, 'out') < 8e-2
    # code_only contract (stage II) returns (logits, lq_feat)
    lo, lq2 = model(x, w=1, adain=True, code_only=True)
    assert torch.equal(lo, logits) and torch.equal(lq2, lq)


def test_vq_path_codes_against_reference_golden(model):
    """TDCRQVAE3.forward path: L2-argmin codes vs the reference's (bf16 encoder => compare where the
    reference margin is not razor thin), and bit-exact vs an fp64 argmin on the kernel's own z_e."""
    from oracle.make_golden import golden_input
    from oracle import pgt_oracle as O
    g = load_golden('pgtformer_ref_b1_128_seed1.pt')
    x = golden_input(g['seed'], g['b'], g['H']).to(DEV)
    z_q, loss, codes = model.forward_vq(x, code_only=True)
    assert codes.shape == g['vq_codes'].shape and codes.dtype == torch.int64
    agree = (codes.cpu() == g['vq_codes']).float().mean().item()
    print('L2-argmin code agreement vs reference: %.4f' % agree)
    assert agree > 0.9
    out, _, codes2 = model.forward_vq(x)
    assert torch.equal(codes, codes2) and tuple(out.shape) == tuple(g['vq_out_shape'])


def test_batch_equals_per_clip(model):
    """Clips are independent (SURVEY F5): a b=2 forward equals two b=1 forwards.  Bit-identity across batch sizes is
    asserted for the encoder output (lq_feat) and for the decoder output under forced codes; the logits, which also
    depend on the parsing branch (tiny feature maps whose tile / frame alignment changes with the batch), are compared
    with a tolerance."""
    x = torch.rand(6, 3, 64, 64, generator=torch.Generator().manual_seed(11)).to(DEV)
    lo, lq = model(x, w=1, adain=True, code_only=True)
    lo0, lq0 = model(x[:3], w=1, adain=True, code_only=True)
    lo1, lq1 = model(x[3:], w=1, adain=True, code_only=True)
    assert torch.equal(lq, torch.cat([lq0, lq1], 0))          # encoder path: our kernels only
    assert relerr(lo, torch.cat([lo0, lo1], 0)) < 5e-3
    codes = lo.argmax(-1)
    out = model(x, w=1, adain=True, force_codes=codes)[0]
    out0 = model(x[:3], w=1, adain=True, force_codes=codes[:3])[0]
    out1 = model(x[3:], w=1, adain=True, force_codes=codes[3:])[0]
    assert torch.equal(out, torch.cat([out0, out1], 0))


def test_cuda_graph_replay_matches_eager(model):
    x = torch.rand(3, 3, 128, 128, generator=torch.Generator().manual_seed(12)).to(DEV)
    ref = [t.clone() for t in model(x, w=1, adain=True)]
    model.cuda_graph = True
    try:
        for _ in range(2):
            got = model(x, w=1, adain=True)
            for a, b in zip(got, ref):
                assert torch.equal(a, b)
        x2 = torch.rand(3, 3, 128, 128, generator=torch.Generator().manual_seed(13)).to(DEV)
        got2 = [t.clone() for t in model(x2, w=1, adain=True)]
    finally:
        model.cuda_graph = False
    ref2 = model(x2, w=1, adain=True)
    for a, b in zip(got2, ref2):
        assert torch.equal(a, b)


def _record(name, res):
    """Prints the measured parity numbers with the test output."""
    import json
    print('parity[%s] %s' % (name, json.dumps(res)))


@pytest.mark.parametrize('size', [512, 1024])
def test_forward_against_reference_golden_full_size(model, size):
    """The BASELINE sizes against outputs of the reference itself: 512^2 is the UNPATCHED reference's native size
    (`README.md:93`), 1024^2 the reference with the three size patches of oracle/reference_loader.py.  The fixture
    keeps every code index and top-2 logit margin, sampled logit rows, lq_feat (fp16) and the middle output frame
    (oracle/make_golden.py --full).  Bounds: the measured values of this kernel set with a small margin (512^2:
    lq 1.6e-2, logits 1.0e-2, agreement 0.941, teacher-forced PSNR 37.6 dB).  The synthetic checkpoint's top-1 / top-2
    logit margins are tiny (median 0.05, 10 % below 0.012), so bf16 activations flip near-ties: tools/
    diag_code_agreement.py attributes 3.4 points to the bf16 encoder activations (lq_feat mean error 2e-3, the same as
    the reference's own bf16 autocast, SURVEY F9) and 0.8 to the bf16 operands of the global transformer; wherever the
    reference's margin exceeds 3x the measured logit error the codes agree exactly (code_agree_confident)."""
    import sys
    import os
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tools'))
    from parity_check import check_compact
    res = check_compact(model, size, DEV)
    _record('golden_%d' % size, res)
    assert res['lq_rel'] < 2.5e-2 and res['logits_rel'] < 2e-2
    assert res['code_agree'] > 0.92, res
    assert res['code_agree_confident'] > 0.999, res          # a flip where the reference is decisive is a kernel error
    assert res['psnr_tf'] > 36.5 and res['out_tf_rel'] < 6e-2, res
    assert res['vq_code_agree'] > 0.985, res


def test_demo_video_psnr_against_reference(model):
    """First 8 frames of the reference's assets/inputdemovideo.mp4 (downscaled to 128^2) through the streaming pipeline
    vs the reference's own `inference.py` loop on the same frames (fixture: oracle/make_golden.py --video), same
    synthetic checkpoint."""
    import sys
    import os
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tools'))
    from parity_check import check_demo_video
    res = check_demo_video(model)
    _record('demo_video', res)
    # measured: delta 0.040 dB, direct PSNR 21.8 dB — the ~6 % near-tie code flips of the synthetic checkpoint change
    # whole 16x16 patches; with decisive logits (trained weights) the two restorations coincide
    assert abs(res['psnr_delta_db']) < 0.08, res
    assert res['psnr_vs_reference'] > 20.0, res


@pytest.mark.parametrize('size,clips', [(512, 2), (1024, 1)])
def test_full_size_properties(model, size, clips):
    """Size-independent properties at the BASELINE sizes, b > 1 (the comparison with the reference's own outputs at
    these sizes is test_forward_against_reference_golden_full_size) — determinism, clip independence (a clip's result does not depend
    on its batch neighbours), code indices in range, finite outputs in a sane range."""
    g = torch.Generator().manual_seed(40 + size)
    x = torch.rand(clips * 3, 3, size, size, generator=g).to(DEV)
    out, logits, lq = [t.clone() for t in model(x, w=1, adain=True)]
    hh = size // 16
    assert out.shape == (clips * 3, 3, size, size) and logits.shape == (clips * 3, hh, hh, 1, 1024) and lq.shape == (clips * 3, hh, hh, 512)
    for t in (out, logits, lq):
        assert torch.isfinite(t).all()
    assert out.abs().max().item() < 50
    codes = model.engine().last_codes
    assert codes.min().item() >= 0 and codes.max().item() < 1024
    again = model(x, w=1, adain=True)
    assert torch.equal(again[0], out) and torch.equal(again[1], logits)          # deterministic
    first = model(x[:3].contiguous(), w=1, adain=True)
    assert torch.equal(first[0], out[:3]) and torch.equal(first[2], lq[:3])      # clip 0 alone == clip 0 in the batch
