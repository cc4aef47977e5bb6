"""GPU parity tests, kernel by kernel, THROUGH THE C ABI (pgtformer_b200.ops -> ctypes ->
libpgt_b200.so) against the CPU oracle (oracle/pgt_oracle.py) on identical bf16-rounded
inputs.  Tolerances (SURVEY F9): fp32-output epilogues are compared at 1e-3 * max|ref|;
bf16 outputs at one bf16 ulp of the oracle value (+ the same absolute floor); index outputs
bit-exact.  Where `rel` is larger than 1e-3 the kernel rounds an INTERMEDIATE to bf16 that the fp32 oracle does not —
each such test says which one:
  * attention kernels (window, MHA), 4e-3: the softmax probabilities P are bf16 operands of the P V tensor-core product
    (relative rounding 2^-9 per element of a convex combination);
  * fused Swin MLP, 4e-3: the GELU(fc1) hidden tile is a bf16 operand of fc2; fused LN + linear, 3e-3: LN(x) is a bf16
    operand of the projection; their folded-affine variants (gamma / beta inside the weights), 4e-3 / 6e-3 against the
    fp32 block with UNROUNDED weights: W * gamma is rounded to bf16 once on top of the above;
  * upsample-folded conv, 6e-3: each 2x2 phase weight is a SUM of up to four 3x3 taps rounded to bf16 once (the oracle
    multiplies the four bf16 taps separately); RGB stem with normalisation, 6e-3: the normalised pixel is rounded to bf16;
  * GroupNorm from fused statistics, 3e-3: the statistics are accumulated from the producer's fp32 accumulators, the
    oracle's from the bf16-rounded tensor the apply pass then normalises."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = 'cuda'


def ops():
    from pgtformer_b200 import ops as o
    return o


def bf(x):
    return x.to(torch.bfloat16)


def rnd(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g) * scale


def check_close(got, ref, what, bf16_out=False, rel=1e-3):
    got = got.float().cpu()
    ref = ref.float().cpu()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert torch.isfinite(got).all(), what + ': non-finite output'
    mx = ref.abs().max().item()
    err = (got - ref).abs()
    if bf16_out:
        tol = ref.abs() * 2.0 ** -8 + rel * mx
        bad = (err > tol)
        assert not bad.any(), '%s: %d elements beyond 1 bf16 ulp (max err %.3e, max|ref| %.3e)' % (
            what, int(bad.sum()), err.max().item(), mx)
    else:
        assert err.max().item() <= rel * mx, '%s: max err %.3e > %.1e * max|ref| %.3e' % (what, err.max().item(), rel, mx)


def pack_conv_weight(w):
    """OIHW fp32 -> [Cout, k*k*CinPad] bf16, K index = tap*CinPad + c (see include/pgt_b200.h)."""
    co, ci, kh, kw = w.shape
    cp = (ci + 63) // 64 * 64
    wp = torch.zeros(co, kh * kw, cp)
    wp[:, :, :ci] = w.permute(0, 2, 3, 1).reshape(co, kh * kw, ci)
    return bf(wp.reshape(co, kh * kw * cp)).contiguous()


# ------------------------------------------------------------------------------------ GEMM
@pytest.mark.parametrize('M,N,K,act,res,out_dt', [
    (300, 96, 192, 'gelu', True, torch.float32),
    (1024, 768, 256, None, False, torch.bfloat16),
    (130, 1024, 512, None, False, torch.float32),
    (4096, 256, 256, None, True, torch.bfloat16),
    (257, 32, 512, 'silu', False, torch.float32),
    (20000, 512, 1024, None, False, torch.float32),
    (192, 1536, 512, None, False, torch.bfloat16),
])
def test_linear(M, N, K, act, res, out_dt):
    o = ops()
    a, w, b = bf(rnd((M, K), 1)), bf(rnd((N, K), 2, K ** -0.5)), rnd((N,), 3, 0.1)
    r = bf(rnd((M, N), 4)) if res else None
    ref = a.float() @ w.float().t() + b
    if act == 'gelu':
        ref = F.gelu(ref)
    elif act == 'silu':
        ref = F.silu(ref)
    if res:
        ref = ref + r.float()
    out = torch.empty(M, N, dtype=out_dt, device=DEV)
    actc = {None: o.ACT_NONE, 'gelu': o.ACT_GELU, 'silu': o.ACT_SILU}[act]
    o.linear(a.to(DEV), w.to(DEV), out, bias=b.to(DEV), act=actc, residual=r.to(DEV) if res else None)
    torch.cuda.synchronize()
    check_close(out, ref, 'linear', bf16_out=(out_dt == torch.bfloat16))


@pytest.mark.parametrize('M,N,K', [(1000, 512, 512), (3072, 1024, 512), (130, 96, 64)])
def test_linear_fp32_residual_stream(M, N, K):
    """fp32 residual + fp32 output (global transformer): residual TMA-loaded into the staging slot."""
    o = ops()
    a, w, b = bf(rnd((M, K), 1)), bf(rnd((N, K), 2, K ** -0.5)), rnd((N,), 3, 0.1)
    r = rnd((M, N), 4)
    out = torch.empty(M, N, dtype=torch.float32, device=DEV)
    o.linear(a.to(DEV), w.to(DEV), out, bias=b.to(DEV), residual=r.to(DEV))
    torch.cuda.synchronize()
    check_close(out, a.float() @ w.float().t() + b + r, 'linear fp32 residual')
    # in-place residual stream (out aliases residual), as the engine may do
    rr = r.to(DEV).clone()
    o.linear(a.to(DEV), w.to(DEV), rr, bias=b.to(DEV), residual=rr)
    torch.cuda.synchronize()
    check_close(rr, a.float() @ w.float().t() + b + r, 'linear in-place residual')


def test_linear_k_tail_and_strided_views():
    """K = 57 (convpos) inside a 64-wide buffer; output into a channel slice of a wider buffer."""
    o = ops()
    M, N, K = 200, 512, 57
    a_full = torch.zeros(M, 64)
    a_full[:, :K] = rnd((M, K), 5)
    w_full = torch.zeros(N, 64)
    w_full[:, :K] = rnd((N, K), 6, 0.1)
    a, w = bf(a_full).to(DEV), bf(w_full).to(DEV)
    buf = torch.zeros(M, 1056, dtype=torch.bfloat16, device=DEV)
    o.linear(a, w, buf[:, 512:1024], K=K)
    torch.cuda.synchronize()
    ref = bf(a_full).float() @ bf(w_full).float().t()
    check_close(buf[:, 512:1024], ref, 'linear k-tail', bf16_out=True)
    assert buf[:, :512].abs().max() == 0 and buf[:, 1024:].abs().max() == 0


# ------------------------------------------------------------------------------------ conv
def conv_ref(x_nhwc, w, b, stride=1, pad=(1, 1, 1, 1)):
    x = x_nhwc.float().permute(0, 3, 1, 2)
    return F.conv2d(F.pad(x, pad), w, b, stride=stride).permute(0, 2, 3, 1)


@pytest.mark.parametrize('Fr,H,W,Cin,Cout', [
    (3, 16, 16, 64, 64),
    (3, 8, 8, 512, 512),       # two frames per 128-row tile, odd frame count
    (6, 32, 32, 256, 128),
    (3, 8, 128, 128, 64),      # one image row per tile
    (3, 16, 16, 288, 128),     # Cin = 4.5 x 64: channel tail zero-filled by TMA
    (2, 64, 64, 64, 96),
    (3, 4, 4, 64, 64),
    (3, 24, 40, 64, 128),      # halo tiles (8x16) with ragged bottom / right edges
    (1, 8, 16, 128, 32),
])
def test_conv3x3(Fr, H, W, Cin, Cout):
    o = ops()
    x = bf(rnd((Fr, H, W, Cin), 10))
    w = bf(rnd((Cout, Cin, 3, 3), 11, (9 * Cin) ** -0.5)).float()
    b = rnd((Cout,), 12, 0.1)
    out = torch.empty(Fr, H, W, Cout, dtype=torch.float32, device=DEV)
    o.conv(x.to(DEV), pack_conv_weight(w).to(DEV), Cout, out, bias=b.to(DEV))
    torch.cuda.synchronize()
    check_close(out, conv_ref(x, w, b), 'conv3x3')


def test_conv3x3_epilogues_and_nchw():
    o = ops()
    Fr, H, W, C = 3, 16, 16, 128
    x = bf(rnd((Fr, H, W, C), 20))
    w = bf(rnd((C, C, 3, 3), 21, (9 * C) ** -0.5)).float()
    b = rnd((C,), 22, 0.1)
    res, scale = bf(rnd((Fr, H, W, C), 23)), bf(rnd((Fr, H, W, C), 24))
    wp = pack_conv_weight(w).to(DEV)
    y = conv_ref(x, w, b)
    out = torch.empty(Fr, H, W, C, dtype=torch.bfloat16, device=DEV)
    o.conv(x.to(DEV), wp, C, out, bias=b.to(DEV), act=o.ACT_LRELU02)
    check_close(out, F.leaky_relu(y, 0.2), 'conv+lrelu', bf16_out=True)
    o.conv(x.to(DEV), wp, C, out, bias=b.to(DEV), residual=res.to(DEV))
    check_close(out, y + res.float(), 'conv+residual', bf16_out=True)
    o.conv(x.to(DEV), wp, C, out, bias=b.to(DEV), residual=res.to(DEV), sft_scale=scale.to(DEV), sft_w=0.7)
    check_close(out, res.float() + 0.7 * (res.float() * scale.float() + y), 'conv+sft', bf16_out=True)
    # Cout = 3, fp32 NCHW output (decoder.conv_out)
    w3 = bf(rnd((3, C, 3, 3), 25, (9 * C) ** -0.5)).float()
    b3 = rnd((3,), 26, 0.1)
    out3 = torch.empty(Fr, 3, H, W, dtype=torch.float32, device=DEV)
    o.conv(x.to(DEV), pack_conv_weight(w3).to(DEV), 3, out3, bias=b3.to(DEV), nchw=True)
    check_close(out3, conv_ref(x, w3, b3).permute(0, 3, 1, 2), 'conv nchw')


@pytest.mark.parametrize('Fr,H,W,C,pad_lo', [(3, 16, 16, 64, 0), (3, 32, 32, 128, 0), (3, 16, 16, 64, 1), (6, 8, 8, 256, 1)])
def test_conv3x3_stride2(Fr, H, W, C, pad_lo):
    """pad_lo=0: Downsample pad(0,1,0,1) (tdcrqvae3_arch.py:67-76); pad_lo=1: ResNet 3x3 s2 p1."""
    o = ops()
    x = bf(rnd((Fr, H, W, C), 30))
    w = bf(rnd((C, C, 3, 3), 31, (9 * C) ** -0.5)).float()
    b = rnd((C,), 32, 0.1)
    out = torch.empty(Fr, H // 2, W // 2, C, dtype=torch.float32, device=DEV)
    o.conv(x.to(DEV), pack_conv_weight(w).to(DEV), C, out, stride=2, pad_lo=pad_lo, bias=b.to(DEV))
    torch.cuda.synchronize()
    pad = (0, 1, 0, 1) if pad_lo == 0 else (1, 1, 1, 1)
    check_close(out, conv_ref(x, w, b, stride=2, pad=pad), 'conv s2')


def test_conv1x1_stride2():
    o = ops()
    Fr, H, W, Cin, Cout = 3, 16, 16, 64, 128
    x = bf(rnd((Fr, H, W, Cin), 33))
    w = bf(rnd((Cout, Cin, 1, 1), 34, Cin ** -0.5)).float()
    out = torch.empty(Fr, H // 2, W // 2, Cout, dtype=torch.float32, device=DEV)
    o.conv(x.to(DEV), pack_conv_weight(w).to(DEV), Cout, out, ksize=1, stride=2, pad_lo=0)
    check_close(out, conv_ref(x, w, None, stride=2, pad=(0, 0, 0, 0)), 'conv1x1 s2')


@pytest.mark.parametrize('Fr,H,W,C', [(3, 8, 8, 64), (3, 16, 16, 128), (2, 4, 4, 512), (3, 32, 32, 256), (2, 40, 20, 64),
                                      (2, 32, 24, 96)])
def test_conv_up2x_folded(Fr, H, W, C):
    """nearest x2 + conv3x3 (tdcrqvae3_arch.py:45-52) as four 2x2 phase convs on the source resolution."""
    from pgtformer_b200.engine import _pack_up2x
    o = ops()
    x = bf(rnd((Fr, H, W, C), 35))
    w = bf(rnd((C, C, 3, 3), 36, (9 * C) ** -0.5)).float()
    b = rnd((C,), 37, 0.1)
    out = torch.empty(Fr, 2 * H, 2 * W, C, dtype=torch.bfloat16, device=DEV)
    o.conv_up2x(x.to(DEV), _pack_up2x(w.to(DEV)), C, out, bias=b.to(DEV))
    torch.cuda.synchronize()
    up = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2.0, mode='nearest')
    ref = F.conv2d(up, w, b, padding=1).permute(0, 2, 3, 1)
    # tap-summed weights are rounded to bf16 once more: allow 2 ulp
    check_close(out, ref, 'conv up2x', bf16_out=True, rel=6e-3)


# ------------------------------------------------------------------------------------ norms
@pytest.mark.parametrize('Fr,HW,C', [(3, 64, 64), (3, 1024, 512), (2, 4096, 128), (3, 256, 1056), (3, 1024, 288), (3, 64, 544)])
def test_groupnorm_silu(Fr, HW, C):
    o = ops()
    x = bf(rnd((Fr, HW, C), 50) * 2 + 0.3)
    gam, bet = 1 + 0.1 * rnd((C,), 51), 0.1 * rnd((C,), 52)
    out = torch.empty(Fr, HW, C, dtype=torch.bfloat16, device=DEV)
    o.groupnorm_silu(x.to(DEV), gam.to(DEV), bet.to(DEV), out)
    ref = F.silu(F.group_norm(x.float().permute(0, 2, 1), 32, gam, bet, eps=1e-6)).permute(0, 2, 1)
    check_close(out, ref, 'groupnorm+silu', bf16_out=True)
    o.groupnorm_silu(x.to(DEV), gam.to(DEV), bet.to(DEV), out, silu=False)
    check_close(out, F.group_norm(x.float().permute(0, 2, 1), 32, gam, bet, eps=1e-6).permute(0, 2, 1), 'groupnorm', bf16_out=True)


@pytest.mark.parametrize('T,C,dt', [(1000, 256, torch.bfloat16), (3072, 512, torch.bfloat16), (77, 512, torch.float32)])
def test_layernorm(T, C, dt):
    o = ops()
    x = (rnd((T, C), 60) * 1.5 + 0.2).to(dt)
    gam, bet = 1 + 0.1 * rnd((C,), 61), 0.1 * rnd((C,), 62)
    pos = bf(rnd((T, C), 63))
    y = torch.empty(T, C, dtype=torch.bfloat16, device=DEV)
    y2 = torch.empty_like(y)
    o.layernorm(x.to(DEV), gam.to(DEV), bet.to(DEV), y, pos=pos.to(DEV), out2=y2)
    ref = F.layer_norm(x.float(), (C,), gam, bet, 1e-5)
    check_close(y, ref, 'layernorm', bf16_out=True)
    check_close(y2, ref + pos.float(), 'layernorm+pos', bf16_out=True)


def test_adain():
    from oracle import pgt_oracle as O
    o = ops()
    Fr, HW, C = 3, 64, 512
    q, l = rnd((Fr, HW, C), 70), bf(rnd((Fr, HW, C), 71) * 0.5 + 0.1)
    out = torch.empty(Fr, HW, C, dtype=torch.bfloat16, device=DEV)
    o.adain(q.to(DEV), l.to(DEV), out)
    ref = O.adain(q.permute(0, 2, 1).reshape(Fr, C, 8, 8), l.float().permute(0, 2, 1).reshape(Fr, C, 8, 8))
    check_close(out, ref.reshape(Fr, C, HW).permute(0, 2, 1), 'adain', bf16_out=True)


# ------------------------------------------------------------------------------------ codebook
def test_argmax_gather_bit_exact(synth_sd):
    from oracle import pgt_oracle as O
    o = ops()
    cb = synth_sd['quantizer.codebooks.0.weight']
    T, K = 3 * 64 + 5, 1024
    logits = rnd((T, K), 80)
    logits[0, 17] = logits[0].max() + 1
    logits[0, 900] = logits[0, 17]              # duplicate maximum -> first index wins
    logits[1, :] = 0.25                         # all ties -> index 0
    idx = torch.empty(T, dtype=torch.int64, device=DEV)
    quant = torch.empty(T, 512, dtype=torch.float32, device=DEV)
    o.argmax_gather(logits.to(DEV), cb.to(DEV), idx, quant)
    ref_idx = logits.argmax(-1)
    assert torch.equal(idx.cpu(), ref_idx)
    assert idx[0] == 17 and idx[1] == 0
    assert torch.equal(quant.cpu(), O.embed_code(cb, ref_idx.view(T, 1)))
    qb = torch.empty(T, 512, dtype=torch.bfloat16, device=DEV)
    forced = torch.randint(0, 1024, (T,), generator=torch.Generator().manual_seed(81))
    o.argmax_gather(logits.to(DEV), cb.to(DEV), idx, qb, idx_in=forced.to(DEV))
    assert torch.equal(idx.cpu(), forced) and torch.equal(qb.cpu(), bf(cb[forced]))


@pytest.mark.parametrize('regime', ['random', 'near_code', 'duplicates'])
def test_l2_argmin_bit_exact(synth_sd, regime):
    from oracle import pgt_oracle as O
    o = ops()
    cb = synth_sd['quantizer.codebooks.0.weight'].clone()
    T = 3 * 8 * 8 * 4 + 7
    if regime == 'random':
        z = rnd((T, 512), 90)
    elif regime == 'near_code':
        pick = torch.randint(0, 1024, (T,), generator=torch.Generator().manual_seed(91))
        z = cb[pick] + 0.05 * rnd((T, 512), 92)
    else:
        cb[700] = cb[3]
        cb[701] = cb[3]
        z = cb[3].expand(T, 512) + 0.01 * rnd((T, 512), 93)
    idx = torch.empty(T, dtype=torch.int64, device=DEV)
    quant = torch.empty(T, 512, dtype=torch.float32, device=DEV)
    o.l2_argmin(z.to(DEV).contiguous(), cb.to(DEV).contiguous(), 1024, idx, quant)
    ref, _ = O.l2_argmin_exact(cb, z)
    assert torch.equal(idx.cpu(), ref), 'mismatches: %d' % int((idx.cpu() != ref).sum())
    assert torch.equal(quant.cpu(), cb[ref])
    assert int(idx.max()) < 1024
    if regime == 'duplicates':
        assert (idx.cpu() == 3).all()
    # the reference's own fp32 addmm formula agrees wherever its margin is meaningful
    ref32 = O.l2_argmin(cb, z)
    assert (ref32 == ref).float().mean() > 0.995


# ------------------------------------------------------------------------------------ attention
@pytest.mark.parametrize('C,H,W,clips', [(256, 16, 16, 1), (512, 8, 8, 2), (256, 32, 32, 1), (512, 4, 4, 1)])
@pytest.mark.parametrize('shifted', [False, True])
def test_window_attention_core(C, H, W, clips, shifted):
    """Core only (q/kv/proj identity): compares against the oracle's roll/partition/attention/reverse."""
    from oracle import pgt_oracle as O
    from pgtformer_b200.weights import relative_position_index
    o = ops()
    heads, d = 8, C // 8
    T = clips * 3 * H * W
    qkv = bf(rnd((T, 3 * C), 100, 1.0))
    table = 0.5 * rnd((245, heads), 101)
    idx = relative_position_index()
    bias_tab = table[idx.view(-1)].view(48, 48, heads).permute(2, 0, 1).contiguous()
    out = torch.empty(T, C, dtype=torch.bfloat16, device=DEV)
    o.window_attention(qkv.to(DEV), clips, H, W, C, heads, 2 if shifted else 0, bias_tab.to(DEV), out)
    torch.cuda.synchronize()
    # oracle: feed q, k, v through identity projections
    x = qkv.float().view(clips, 3, H, W, 3 * C)
    do_shift = shifted and H > 4 and W > 4
    xs = torch.roll(x, (-2, -2), (2, 3)) if do_shift else x
    xw = O.window_partition(xs).view(-1, 48, 3 * C)
    q = xw[..., :C].view(-1, 48, heads, d).permute(0, 2, 1, 3) * d ** -0.5
    k = xw[..., C:2 * C].view(-1, 48, heads, d).permute(0, 2, 1, 3)
    v = xw[..., 2 * C:].view(-1, 48, heads, d).permute(0, 2, 1, 3)
    attn = q @ k.transpose(-2, -1) + bias_tab[None]
    if do_shift:
        mask = O.shift_mask(H, W)
        nW = mask.shape[0]
        attn = (attn.view(-1, nW, heads, 48, 48) + mask[None, :, None]).view(-1, heads, 48, 48)
    ow = (attn.softmax(-1) @ v).transpose(1, 2).reshape(-1, 48, C)
    ref = O.window_reverse(ow.view(-1, 3, 4, 4, C), clips, 3, H, W)
    if do_shift:
        ref = torch.roll(ref, (2, 2), (2, 3))
    check_close(out, ref.reshape(T, C), 'window attention', bf16_out=True, rel=4e-3)


@pytest.mark.parametrize('L,clips', [(192, 2), (3072, 1), (48, 1), (200, 1), (768, 2), (256, 3)])
def test_mha_fwd(L, clips):
    o = ops()
    heads, d, E = 8, 64, 512
    q, k, v = bf(rnd((clips * L, E), 110)), bf(rnd((clips * L, E), 111)), bf(rnd((clips * L, E), 112))
    out = torch.empty(clips * L, E, dtype=torch.bfloat16, device=DEV)
    o.mha(q.to(DEV), k.to(DEV), v.to(DEV), clips, L, heads, d, out)
    torch.cuda.synchronize()
    sh = lambda a: a.float().view(clips, L, heads, d).permute(0, 2, 1, 3)
    ref = (torch.softmax(sh(q) @ sh(k).transpose(-1, -2) / math.sqrt(d), -1) @ sh(v)).permute(0, 2, 1, 3).reshape(clips * L, E)
    check_close(out, ref, 'mha', bf16_out=True, rel=4e-3)


# ------------------------------------------------------------------------------------ layout
def test_layout_kernels():
    o = ops()
    x = torch.rand(3, 3, 16, 16, generator=torch.Generator().manual_seed(120))
    mean, std = torch.tensor([0.485, 0.456, 0.406]), torch.tensor([0.229, 0.224, 0.225])
    y = torch.zeros(3, 16, 16, 8, dtype=torch.bfloat16, device=DEV)
    o.nchw_to_nhwc(x.to(DEV), y, mean.to(DEV), std.to(DEV))
    ref = ((x - mean.view(1, 3, 1, 1)) / std.view(1, 3, 1, 1)).permute(0, 2, 3, 1)
    check_close(y[..., :3], ref, 'nchw->nhwc', bf16_out=True)
    assert y[..., 3:].abs().max() == 0
    a = bf(rnd((2, 8, 8, 64), 121))
    buf = torch.zeros(2, 8, 8, 160, dtype=torch.bfloat16, device=DEV)
    o.copy2d(a.to(DEV), buf[..., 64:128])
    assert torch.equal(buf[..., 64:128].cpu(), a) and buf[..., :64].abs().max() == 0
    f32 = torch.empty(2, 64, 8, 8, dtype=torch.float32, device=DEV)
    o.nhwc_to_f32(a.to(DEV), f32, True)
    assert torch.equal(f32.cpu(), a.float().permute(0, 3, 1, 2))
    f32b = torch.empty(2, 8, 8, 64, dtype=torch.float32, device=DEV)
    o.nhwc_to_f32(a.to(DEV), f32b, False)
    assert torch.equal(f32b.cpu(), a.float())


# ------------------------------------------------------------------------------------ parsing-branch kernels
def test_maxpool_avgpool_affine_assemble():
    o = ops()
    Fr, H, W = 3, 64, 64
    y = bf(rnd((Fr, H // 2, W // 2, 64), 130)).to(DEV)
    mp = torch.empty(Fr, H // 4, W // 4, 64, dtype=torch.bfloat16, device=DEV)
    o.maxpool3x3s2(y, mp)
    refmp = F.max_pool2d(y.float().cpu().permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
    assert torch.equal(mp.float().cpu(), refmp)
    ap = torch.empty(Fr, 64, dtype=torch.bfloat16, device=DEV)
    o.global_avgpool(mp, ap)
    check_close(ap, refmp.mean((1, 2)), 'avgpool', bf16_out=True)
    sc, av = bf(rnd((Fr, 64), 133)), bf(rnd((Fr, 64), 134))
    am = bf(rnd((Fr, H // 4, W // 4, 64), 135))
    out = torch.empty_like(mp)
    o.channel_affine(mp, sc.to(DEV), out, plus_one=True, addv=av.to(DEV), addm=am.to(DEV))
    refa = refmp * (sc.float()[:, None, None, :] + 1) + av.float()[:, None, None, :] + am.float()
    check_close(out, refa, 'channel_affine', bf16_out=True)
    o0, o1 = bf(rnd((Fr, 16, 16, 32), 136)), bf(rnd((Fr, 16, 16, 32), 137))
    o2 = bf(rnd((Fr, 8, 8, 32), 138))
    cond = torch.empty(Fr, 8, 8, 64, dtype=torch.bfloat16, device=DEV)
    o.assemble_cond(o0.to(DEV), o1.to(DEV), o2.to(DEV), cond)
    up = lambda t: F.interpolate(t.float()[..., :19].permute(0, 3, 1, 2), (8, 8), mode='bilinear', align_corners=True).permute(0, 2, 3, 1)
    refc = torch.cat([up(o0), up(o1), o2.float()[..., :19], torch.zeros(Fr, 8, 8, 7)], -1)
    check_close(cond, refc, 'assemble_cond', bf16_out=True)


def test_conv_relu_after_residual():
    o = ops()
    Fr, H, W, C = 3, 16, 16, 256
    x = bf(rnd((Fr, H, W, C), 140))
    w = bf(rnd((C, C, 3, 3), 141, (9 * C) ** -0.5)).float()
    b = rnd((C,), 142, 0.1)
    res = bf(rnd((Fr, H, W, C), 143))
    out = torch.empty(Fr, H, W, C, dtype=torch.bfloat16, device=DEV)
    o.conv(x.to(DEV), pack_conv_weight(w).to(DEV), C, out, bias=b.to(DEV), act=o.ACT_RELU, residual=res.to(DEV),
           relu_after_res=True)
    check_close(out, F.relu(conv_ref(x, w, b) + res.float()), 'conv relu-after-residual', bf16_out=True)


@pytest.mark.parametrize('Fr,H,W,Cin,Cout,lin', [(3, 16, 16, 64, 64, False), (3, 32, 32, 128, 256, False),
                                                (6, 16, 16, 256, 512, False), (3, 16, 32, 64, 128, False),
                                                (3, 16, 16, 256, 256, True)])
def test_groupnorm_stats_fused_in_epilogue(Fr, H, W, Cin, Cout, lin):
    """conv / linear epilogue emits per-tile (sum, sumsq) per GroupNorm group; finalize+apply consumes them."""
    o = ops()
    x = bf(rnd((Fr, H, W, Cin), 150))
    gam, bet = 1 + 0.1 * rnd((Cout,), 153), 0.1 * rnd((Cout,), 154)
    res = bf(rnd((Fr, H, W, Cout), 155))
    y = torch.empty(Fr, H, W, Cout, dtype=torch.bfloat16, device=DEV)
    if lin:
        w = bf(rnd((Cout, Cin), 151, Cin ** -0.5))
        b = rnd((Cout,), 152, 0.1)
        tpf = H * W // 128
        stats = torch.zeros(Fr * tpf * 4 * 64, dtype=torch.float32, device=DEV)
        o.linear(x.to(DEV), w.to(DEV), y, bias=b.to(DEV), residual=res.to(DEV), gn_stats=stats)
        ref = x.float() @ w.float().t() + b + res.float()
    else:
        w = bf(rnd((Cout, Cin, 3, 3), 151, (9 * Cin) ** -0.5)).float()
        b = rnd((Cout,), 152, 0.1)
        tpf = o.conv_tiles_per_frame(H, W, Cout)
        assert tpf > 0
        stats = torch.zeros(Fr * tpf * 4 * 64, dtype=torch.float32, device=DEV)
        o.conv(x.to(DEV), pack_conv_weight(w).to(DEV), Cout, y, bias=b.to(DEV), residual=res.to(DEV), gn_stats=stats)
        ref = conv_ref(x, w, b) + res.float()
    check_close(y, ref, 'producer', bf16_out=True)
    out = torch.empty_like(y)
    o.groupnorm_apply_stats(y, gam.to(DEV), bet.to(DEV), out, stats, tpf * 4)
    gref = F.silu(F.group_norm(y.float().cpu().permute(0, 3, 1, 2), 32, gam, bet, eps=1e-6)).permute(0, 2, 3, 1)
    check_close(out, gref, 'fused-stats groupnorm', bf16_out=True, rel=3e-3)


@pytest.mark.parametrize('T', [128, 1000, 12288])
def test_swin_mlp_fused(T):
    """out = x + fc2(gelu(fc1(LN(x)))) in one kernel vs the fp32 composition on bf16-rounded operands."""
    o = ops()
    C = 256
    x = bf(rnd((T, C), 160) * 1.5 + 0.1)
    g, b = 1 + 0.1 * rnd((C,), 161), 0.1 * rnd((C,), 162)
    w1, b1 = bf(rnd((C, C), 163, C ** -0.5)), rnd((C,), 164, 0.1)
    w2, b2 = bf(rnd((C, C), 165, C ** -0.5)), rnd((C,), 166, 0.1)
    out = torch.empty(T, C, dtype=torch.bfloat16, device=DEV)
    o.swin_mlp(x.to(DEV), g.to(DEV), b.to(DEV), w1.to(DEV), b1.to(DEV), w2.to(DEV), b2.to(DEV), out)
    torch.cuda.synchronize()
    y = bf(F.layer_norm(x.float(), (C,), g, b, 1e-5)).float()
    hdn = bf(F.gelu(y @ w1.float().t() + b1)).float()
    ref = x.float() + hdn @ w2.float().t() + b2
    check_close(out, ref, 'fused swin mlp', bf16_out=True, rel=4e-3)


@pytest.mark.parametrize('Fr,H,W,C', [(3, 16, 16, 128), (2, 32, 64, 64), (3, 16, 16, 512)])
def test_conv_up2x_groupnorm_stats(Fr, H, W, C):
    """The four phase launches of the upsample conv fill one statistics buffer [frame][phase][tile][quad][32][2]."""
    from pgtformer_b200.engine import _pack_up2x
    o = ops()
    x = bf(rnd((Fr, H, W, C), 170))
    w = bf(rnd((C, C, 3, 3), 171, (9 * C) ** -0.5)).float()
    b = rnd((C,), 172, 0.1)
    gam, bet = 1 + 0.1 * rnd((C,), 173), 0.1 * rnd((C,), 174)
    tpf = o.conv_tiles_per_frame(H, W, C, 2, 1, 1)
    assert tpf > 0
    stats = torch.zeros(Fr * 16 * tpf * 64, dtype=torch.float32, device=DEV)
    y = torch.empty(Fr, 2 * H, 2 * W, C, dtype=torch.bfloat16, device=DEV)
    o.conv_up2x(x.to(DEV), _pack_up2x(w.to(DEV)), C, y, bias=b.to(DEV), gn_stats=stats)
    out = torch.empty_like(y)
    o.groupnorm_apply_stats(y, gam.to(DEV), bet.to(DEV), out, stats, 16 * tpf)
    gref = F.silu(F.group_norm(y.float().cpu().permute(0, 3, 1, 2), 32, gam, bet, eps=1e-6)).permute(0, 2, 3, 1)
    check_close(out, gref, 'up2x fused-stats groupnorm', bf16_out=True, rel=3e-3)


@pytest.mark.parametrize('ks,stride,pad,norm,Fr,H,W', [(3, 1, 1, False, 3, 32, 48), (7, 2, 3, True, 3, 32, 48),
                                                       (3, 1, 1, False, 2, 20, 36), (7, 2, 3, True, 5, 64, 64)])
def test_conv_rgb_tensor_core(ks, stride, pad, norm, Fr, H, W):
    """Cin = 3 convs (encoder conv_in, BiSeNet stem) with the im2col done inside the wgmma kernel; ragged last tile,
    normalisation before the zero padding, fused GroupNorm statistics."""
    from pgtformer_b200.engine import _pack_rgb
    o = ops()
    x = torch.rand(Fr, 3, H, W, generator=torch.Generator().manual_seed(180))
    mean, std = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225)) if norm else (None, None)
    w, b = rnd((64, 3, ks, ks), 181, (3 * ks * ks) ** -0.5), rnd((64,), 182, 0.1)
    Ho, Wo = (H + 2 * pad - ks) // stride + 1, (W + 2 * pad - ks) // stride + 1
    xn = x if not norm else (x - torch.tensor(mean).view(1, 3, 1, 1)) / torch.tensor(std).view(1, 3, 1, 1)
    act = o.ACT_RELU if norm else o.ACT_NONE
    stats = None
    if (Ho * Wo) % 128 == 0:
        stats = torch.zeros(Fr * (Ho * Wo // 128) * 4 * 64, dtype=torch.float32, device=DEV)
    out = torch.empty(Fr, Ho, Wo, 64, dtype=torch.bfloat16, device=DEV)
    o.conv_rgb(x.to(DEV), _pack_rgb(w.to(DEV)), b.to(DEV), out, ks, stride, pad, act=act, mean3=mean, std3=std,
               gn_stats=stats)
    ref = F.conv2d(bf(xn).float(), bf(w).float(), b, stride=stride, padding=pad)
    ref = (F.relu(ref) if norm else ref).permute(0, 2, 3, 1)
    # (x - mean) * (1 / std) may round to the neighbouring bf16 of (x - mean) / std: a hair above pure bf16 output noise
    check_close(out, ref, 'rgb conv', bf16_out=True, rel=6e-3 if norm else 1e-3)
    if stats is not None:
        gam, bet = 1 + 0.1 * rnd((64,), 183), 0.1 * rnd((64,), 184)
        y = torch.empty_like(out)
        o.groupnorm_apply_stats(out, gam.to(DEV), bet.to(DEV), y, stats, (Ho * Wo // 128) * 4)
        gref = F.silu(F.group_norm(out.float().cpu().permute(0, 3, 1, 2), 32, gam, bet, eps=1e-6)).permute(0, 2, 3, 1)
        check_close(y, gref, 'rgb conv fused-stats groupnorm', bf16_out=True, rel=3e-3)


@pytest.mark.parametrize('Fr,H,W,Cin,Cout,res,nchw,fused_stats', [
    (3, 32, 24, 64, 64, True, False, True), (2, 16, 8, 160, 64, False, False, False),
    (3, 40, 20, 128, 128, True, False, False), (2, 32, 32, 288, 128, False, False, True),
    (3, 48, 16, 64, 3, False, True, False)])
def test_conv_with_fused_input_groupnorm(Fr, H, W, Cin, Cout, res, nchw, fused_stats):
    """conv3x3(silu(GroupNorm(x))) with the normalisation applied to the slabs in shared memory must equal the
    two-pass path (GroupNorm+SiLU written to HBM, then the conv) bit for bit: same affine terms, same rounding,
    same MMA order; zero padding and channel padding stay zero."""
    o = ops()
    x = bf(rnd((Fr, H, W, Cin), 190) * 1.3 + 0.2).to(DEV)
    gam, bet = (1 + 0.1 * rnd((Cin,), 191)).to(DEV), (0.1 * rnd((Cin,), 192)).to(DEV)
    w = pack_conv_weight(bf(rnd((Cout, Cin, 3, 3), 193, (9 * Cin) ** -0.5)).float()).to(DEV)
    b = rnd((Cout,), 194, 0.1).to(DEV)
    r = bf(rnd((Fr, H, W, Cout), 195)).to(DEV) if res else None
    if not o.conv_gn_supported(H, W, Cin, Cout):
        pytest.skip('halo-reuse conv disabled (PGT_NO_HALO): the fused-GroupNorm variant does not exist')

    def mk():
        return (torch.empty(Fr, Cout, H, W, dtype=torch.float32, device=DEV) if nchw
                else torch.empty(Fr, H, W, Cout, dtype=torch.bfloat16, device=DEV))
    xn = torch.empty_like(x)
    o.groupnorm_silu(x, gam, bet, xn)
    ref = o.conv(xn, w, Cout, mk(), bias=b, residual=r, nchw=nchw)
    ab = torch.empty(Fr * 2 * Cin, dtype=torch.float32, device=DEV)
    o.groupnorm_ab(x, gam, bet, ab)
    stats = None
    if fused_stats:
        tpf = o.conv_tiles_per_frame(H, W, Cout)
        stats = torch.zeros(Fr * tpf * 4 * 64, dtype=torch.float32, device=DEV)
    got = o.conv_gn(x, ab, w, Cout, mk(), bias=b, residual=r, nchw=nchw, gn_stats=stats)
    torch.cuda.synchronize()
    assert torch.equal(got, ref), 'fused-GN conv differs: max |d| = %g' % (got.float() - ref.float()).abs().max().item()
    # and against the fp32 composition
    xr = F.silu(F.group_norm(x.float().cpu().permute(0, 3, 1, 2), 32, gam.cpu(), bet.cpu(), eps=1e-6))
    wr = bf(rnd((Cout, Cin, 3, 3), 193, (9 * Cin) ** -0.5)).float()
    full = F.conv2d(bf(xr).float(), wr, b.cpu(), padding=1)
    if res:
        full = full + r.float().cpu().permute(0, 3, 1, 2)
    if nchw:
        check_close(got, full, 'fused-GN conv vs fp32', rel=4e-3)
    else:
        check_close(got, full.permute(0, 2, 3, 1), 'fused-GN conv vs fp32', bf16_out=True, rel=4e-3)
    if stats is not None:
        y = torch.empty_like(got)
        g2, b2 = (1 + 0.1 * rnd((Cout,), 196)).to(DEV), (0.1 * rnd((Cout,), 197)).to(DEV)
        o.groupnorm_apply_stats(got, g2, b2, y, stats, tpf * 4)
        gref = F.silu(F.group_norm(got.float().cpu().permute(0, 3, 1, 2), 32, g2.cpu(), b2.cpu(), eps=1e-6)).permute(0, 2, 3, 1)
        check_close(y, gref, 'stats after fused-GN conv', bf16_out=True, rel=3e-3)


@pytest.mark.parametrize('T,N', [(128, 768), (1000, 768), (12288, 256), (5000, 512)])
def test_ln_linear_fused(T, N):
    """out = LN(x) W^T + b in one kernel vs the fp32 composition on bf16-rounded operands."""
    o = ops()
    C = 256
    x = bf(rnd((T, C), 200) * 1.5 + 0.1)
    g, b = 1 + 0.1 * rnd((C,), 201), 0.1 * rnd((C,), 202)
    w, wb = bf(rnd((N, C), 203, C ** -0.5)), rnd((N,), 204, 0.1)
    out = torch.full((T, N), 9.0, dtype=torch.bfloat16, device=DEV)
    o.ln_linear(x.to(DEV), g.to(DEV), b.to(DEV), w.to(DEV), wb.to(DEV), out)
    torch.cuda.synchronize()
    y = bf(F.layer_norm(x.float(), (C,), g, b, 1e-5)).float()
    check_close(out, y @ w.float().t() + wb, 'fused LN + linear', bf16_out=True, rel=3e-3)

@pytest.mark.parametrize('T,N', [(1000, 768), (12288, 256)])
def test_ln_linear_folded_affine(T, N):
    """NULL gamma / beta in the C ABI: the caller folded the LayerNorm affine into the weights (W * gamma, bias + W beta),
    as Engine._repack does for norm1 -> q/kv.  Checked against the fp32 LayerNorm + linear of the UNFOLDED parameters:
    the folded path rounds W * gamma once instead of rounding LN(x) and W separately, same tolerance."""
    o = ops()
    C = 256
    x = bf(rnd((T, C), 210) * 1.5 + 0.1)
    g, b = 1 + 0.1 * rnd((C,), 211), 0.1 * rnd((C,), 212)
    w, wb = rnd((N, C), 213, C ** -0.5), rnd((N,), 214, 0.1)
    wf = bf(w * g[None, :])
    bf_ = wb + w @ b
    out = torch.full((T, N), 9.0, dtype=torch.bfloat16, device=DEV)
    o.ln_linear(x.to(DEV), None, None, wf.to(DEV), bf_.to(DEV), out)
    torch.cuda.synchronize()
    ref = F.layer_norm(x.float(), (C,), g, b, 1e-5) @ w.t() + wb
    check_close(out, ref, 'LN + linear, affine folded into W', bf16_out=True, rel=4e-3)


def test_swin_mlp_folded_affine():
    """NULL gamma / beta: norm2's affine folded into fc1 (Engine._repack); vs the fp32 composition of the unfolded block."""
    o = ops()
    T, C = 1000, 256
    x = bf(rnd((T, C), 220) * 1.5 + 0.1)
    g, b = 1 + 0.1 * rnd((C,), 221), 0.1 * rnd((C,), 222)
    w1, b1 = rnd((C, C), 223, C ** -0.5), rnd((C,), 224, 0.1)
    w2, b2 = bf(rnd((C, C), 225, C ** -0.5)), rnd((C,), 226, 0.1)
    w1f, b1f = bf(w1 * g[None, :]), b1 + w1 @ b
    out = torch.empty(T, C, dtype=torch.bfloat16, device=DEV)
    o.swin_mlp(x.to(DEV), None, None, w1f.to(DEV), b1f.to(DEV), w2.to(DEV), b2.to(DEV), out)
    torch.cuda.synchronize()
    hdn = F.gelu(F.layer_norm(x.float(), (C,), g, b, 1e-5) @ w1.t() + b1)
    ref = x.float() + hdn @ w2.float().t() + b2
    check_close(out, ref, 'Swin MLP, affine folded into fc1', bf16_out=True, rel=6e-3)

