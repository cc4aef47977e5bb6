"""The softmax and normalisation kernels at the input ranges where such kernels go wrong, against an fp64 evaluation of
the reference formula on the same bf16 / fp32 input values (on the device):

  A. score range of the global attention (`ops.mha`): a planted key whose scaled logit q.k d^-1/2 stands Delta above the
     rest of the row, in the first, a middle or the last key tile; two equal spikes in different tiles; a staircase of
     tile maxima 40 apart (the reference exponent is raised over and over); a spike in only some heads; scores ~1e3
     everywhere.  d = 64 on the wgmma kernel (mha_tc, L % 128 == 0) and the mma.sync kernel, d = 256 / 512 on
     attn_wide_kernel;
  B. score range of the window attention kernels: q and k scaled so that the scores reach a few hundred and bias tables
     of std 2, so that the additive {0, -100} shift mask no longer zeroes the masked keys;
  C. mean offsets: rows or groups mu + sigma * n with mu / sigma up to 1024 (fp32 inputs) or 64 (bf16 inputs), and one
     exactly constant row or group (sigma = 0), whose normalised output must be beta.

Each kernel keeps the bound its own parity test documents (tests/test_kernels_gpu.py): attention 4e-3 * max|ref|;
bf16 outputs one bf16 ulp plus 1e-3 * max|ref| (LN + linear 3e-3, MLP 4e-3, their folded-affine variants 4e-3 / 6e-3,
GroupNorm from fused statistics 3e-3, GroupNorm folded into the conv 4e-3); every output must be finite."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = 'cuda'
DELTAS = [10, 60, 90, 200, 1000]
RATIOS_F32 = [0, 8, 64, 256, 1024]
RATIOS_BF16 = [0, 8, 64]


def ops():
    from pgtformer_b200 import ops as o
    return o


def randn(shape, seed, scale=1.0):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64) * scale


def check_attn(got, ref, what, rel=4e-3):
    got = got.double()
    assert torch.isfinite(got).all(), '%s: %d non-finite outputs' % (what, int((~torch.isfinite(got)).sum()))
    mx = ref.abs().max().item()
    err = (got - ref).abs().max().item()
    assert err <= rel * mx, '%s: max err %.3e > %.0e * max|ref| %.3e' % (what, err, rel, mx)


def check_close(got, ref, what, rel=1e-3):
    """bf16 output: within one bf16 ulp of the fp64 reference plus rel * max|ref|."""
    got = got.double()
    ref = ref.to(got.device).double()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert torch.isfinite(got).all(), '%s: %d non-finite outputs' % (what, int((~torch.isfinite(got)).sum()))
    mx = ref.abs().max().item()
    err = (got - ref).abs()
    bad = err > ref.abs() * 2.0 ** -8 + rel * mx
    assert not bad.any(), '%s: %d elements beyond 1 bf16 ulp + %.0e * max|ref| (max err %.3e, max|ref| %.3e)' % (
        what, int(bad.sum()), rel, err.max().item(), mx)


# ==================================================================================================== A. score range
def ref_attn(q, k, v, clips, L, heads, d, chunk=2048):
    """fp64 softmax(q k^T / sqrt(d)) v per (clip, head) on the bf16 values; q / k / v [clips * L, heads * d]."""
    out = torch.empty(clips * L, heads * d, dtype=torch.float64, device=DEV)
    for c in range(clips):
        for h in range(heads):
            rows, cols = slice(c * L, (c + 1) * L), slice(h * d, (h + 1) * d)
            K, V = k[rows, cols].double(), v[rows, cols].double()
            for i in range(0, L, chunk):
                Q = q[c * L + i:c * L + min(i + chunk, L), cols].double()
                out[c * L + i:c * L + min(i + chunk, L), cols] = torch.softmax(Q @ K.t() / math.sqrt(d), -1) @ V
    return out


ALPHA = 8.0          # every query's component along the shared direction e = the first channel of its head


def base_qkv(clips, L, heads, d, seed):
    """q = ALPHA e + n, k = n with k.e = 0, v = n: scaled logits of about N(0, 1) before anything is planted."""
    T = clips * L
    q, k, v = randn((T, heads, d), seed), randn((T, heads, d), seed + 1), randn((T, heads, d), seed + 2)
    q[:, :, 0] = ALPHA
    k[:, :, 0] = 0.0
    return q, k, v


def plant(k, d, clip, L, key, delta, heads=None):
    """Key `key` of clip `clip` gets k.e = beta with ALPHA * beta / sqrt(d) = delta: its scaled logit stands delta above
    the rest of every query's row."""
    k[clip * L + key, slice(None) if heads is None else heads, 0] = delta * math.sqrt(d) / ALPHA


def run_mha(q, k, v, clips, L, heads, d):
    dev = [t.reshape(clips * L, heads * d).to(torch.bfloat16).to(DEV) for t in (q, k, v)]
    out = torch.full((clips * L, heads * d), float('nan'), dtype=torch.bfloat16, device=DEV)
    ops().mha(dev[0], dev[1], dev[2], clips, L, heads, d, out)
    torch.cuda.synchronize()
    return out, dev


def key_at(where, L, tile):
    return {'first': 5, 'middle': (L // tile // 2) * tile + 3, 'last': L - 7}[where]


# (path, clips, L): mha_tc for L % 128 == 0, the mma.sync kernel otherwise
D64_SHAPES = [('tc', 1, 384), ('tc', 1, 3072), ('tc', 2, 768), ('sync', 1, 200), ('sync', 1, 192)]
D64_IDS = ['%s-c%d-L%d' % s for s in D64_SHAPES]


@pytest.mark.parametrize('shape', D64_SHAPES, ids=D64_IDS)
@pytest.mark.parametrize('where', ['first', 'middle', 'last'])
@pytest.mark.parametrize('delta', DELTAS)
def test_d64_spike(shape, where, delta):
    _, clips, L = shape
    heads, d = 8, 64
    q, k, v = base_qkv(clips, L, heads, d, 100 + L)
    key = key_at(where, L, 128)
    for c in range(clips):
        plant(k, d, c, L, key, delta)
    out, (qd, kd, vd) = run_mha(q, k, v, clips, L, heads, d)
    check_attn(out, ref_attn(qd, kd, vd, clips, L, heads, d), 'd=64 %s spike %g at key %d' % (shape, delta, key))


@pytest.mark.parametrize('shape', D64_SHAPES, ids=D64_IDS)
def test_d64_two_equal_spikes(shape):
    """Two identical keys far above the rest, in the first and the last tile: the output is the mean of their V rows."""
    _, clips, L = shape
    heads, d = 8, 64
    q, k, v = base_qkv(clips, L, heads, d, 200 + L)
    a, b = 5, L - 7
    for c in range(clips):
        plant(k, d, c, L, a, 200.0)
        k[c * L + b] = k[c * L + a]
    out, (qd, kd, vd) = run_mha(q, k, v, clips, L, heads, d)
    check_attn(out, ref_attn(qd, kd, vd, clips, L, heads, d), 'd=64 %s two spikes' % (shape,))
    vv = vd.double().view(clips, L, heads * d)
    mean = ((vv[:, a] + vv[:, b]) / 2)[:, None].expand(clips, L, heads * d).reshape(clips * L, heads * d)
    check_attn(out, mean, 'd=64 %s two spikes vs mean of their V rows' % (shape,))


def staircase(k, d, clips, L, tile, step=40.0):
    """Every key of tile t gets a scaled logit 40 t above the base: each tile's maximum is 40 above the previous one."""
    t = (torch.arange(clips * L) % L) // tile
    k[:, :, 0] = (step * math.sqrt(d) / ALPHA) * t.double()[:, None]


@pytest.mark.parametrize('shape', D64_SHAPES, ids=D64_IDS)
def test_d64_staircase(shape):
    _, clips, L = shape
    heads, d = 8, 64
    q, k, v = base_qkv(clips, L, heads, d, 300 + L)
    staircase(k, d, clips, L, 128)
    out, (qd, kd, vd) = run_mha(q, k, v, clips, L, heads, d)
    check_attn(out, ref_attn(qd, kd, vd, clips, L, heads, d), 'd=64 %s staircase' % (shape,))


@pytest.mark.parametrize('shape', D64_SHAPES, ids=D64_IDS)
def test_d64_spike_in_some_heads(shape):
    """A spike planted in heads 1, 4, 6 only: the other heads' outputs are bit-identical to a run without it."""
    _, clips, L = shape
    heads, d = 8, 64
    q, k, v = base_qkv(clips, L, heads, d, 400 + L)
    plain, _ = run_mha(q, k, v, clips, L, heads, d)
    spiked = [1, 4, 6]
    for c in range(clips):
        plant(k, d, c, L, key_at('last', L, 128), 200.0, heads=spiked)
    out, (qd, kd, vd) = run_mha(q, k, v, clips, L, heads, d)
    check_attn(out, ref_attn(qd, kd, vd, clips, L, heads, d), 'd=64 %s spike in some heads' % (shape,))
    for h in range(heads):
        if h not in spiked:
            assert torch.equal(out[:, h * d:(h + 1) * d], plain[:, h * d:(h + 1) * d]), 'head %d changed' % h


@pytest.mark.parametrize('shape', D64_SHAPES, ids=D64_IDS)
def test_d64_large_scores(shape):
    """Scaled logits of magnitude ~1e3 everywhere."""
    _, clips, L = shape
    heads, d = 8, 64
    T = clips * L
    q, k, v = randn((T, heads, d), 500 + L, 18.0), randn((T, heads, d), 501 + L, 18.0), randn((T, heads, d), 502 + L)
    out, (qd, kd, vd) = run_mha(q, k, v, clips, L, heads, d)
    s = (qd[:L, :d].double() @ kd[:L, :d].double().t()) / math.sqrt(d)
    assert s.abs().max().item() > 1e3
    check_attn(out, ref_attn(qd, kd, vd, clips, L, heads, d), 'd=64 %s large scores' % (shape,))


WIDE_TILE = {256: 64, 512: 32}       # keys per K/V tile of attn_wide_kernel


@pytest.mark.parametrize('d', [256, 512])
@pytest.mark.parametrize('L', [1024, 4096])
@pytest.mark.parametrize('where', ['middle', 'last'])
@pytest.mark.parametrize('delta', DELTAS)
def test_wide_spike(d, L, where, delta):
    clips, heads = 1, 2
    q, k, v = base_qkv(clips, L, heads, d, 600 + L)
    plant(k, d, 0, L, key_at(where, L, WIDE_TILE[d]), delta)
    out, (qd, kd, vd) = run_mha(q, k, v, clips, L, heads, d)
    check_attn(out, ref_attn(qd, kd, vd, clips, L, heads, d), 'd=%d L=%d %s spike %g' % (d, L, where, delta))


# With the output carried by the few keys of the last tile, the bf16 rounding of P (2^-9 relative per weight) moves a
# row by up to 2^-9 * max|v - out| rather than averaging out: measured 2.8e-3 to 5e-3 * max|ref| over staircase steps
# of 5 to 40 at d = 512 (no overflow, no lost row).  The bound stays as documented; this seed exceeds it.
WIDE_STAIR_XFAIL = pytest.mark.xfail(strict=True, reason='attn_wide d = 512: bf16 P rounding with few dominant keys, '
                                                         '5e-3 * max|ref| against the 4e-3 bound')


@pytest.mark.parametrize('d,L', [(256, 1024), (256, 4096), (512, 4096), pytest.param(512, 1024, marks=WIDE_STAIR_XFAIL)])
def test_wide_staircase(d, L):
    clips, heads = 1, 2
    q, k, v = base_qkv(clips, L, heads, d, 700 + L)
    staircase(k, d, clips, L, WIDE_TILE[d])
    out, (qd, kd, vd) = run_mha(q, k, v, clips, L, heads, d)
    check_attn(out, ref_attn(qd, kd, vd, clips, L, heads, d), 'd=%d L=%d staircase' % (d, L))


# ==================================================================================================== B. window attention
QK_SCALE = 8.0       # q, k entries of std 8: scaled logits of std 64, maxima of a few hundred
BIAS_STD = 2.0


def window_qkv(T, C, seed):
    x = randn((T, 3 * C), seed)
    x[:, :2 * C] *= QK_SCALE
    return x.to(torch.bfloat16)


def window2d_reference(qkv, clips, H, W, C, heads, bias_tab, shifted):
    """fp64 roll / partition / softmax(q k^T d^-1/2 + bias + {0, -100} mask) v / reverse with the oracle's helpers."""
    from oracle import pgt_oracle as O
    d = C // heads
    x = qkv.double().view(clips, 3, H, W, 3 * C)
    sy, sx = O.window_shift(H, W) if shifted else (0, 0)      # get_window_size: each axis on its own
    do_shift = sy > 0 or sx > 0
    xs = torch.roll(x, (-sy, -sx), (2, 3))
    xw = O.window_partition(xs).reshape(-1, 48, 3 * C)
    q = xw[..., :C].reshape(-1, 48, heads, d).permute(0, 2, 1, 3) * d ** -0.5
    k = xw[..., C:2 * C].reshape(-1, 48, heads, d).permute(0, 2, 1, 3)
    v = xw[..., 2 * C:].reshape(-1, 48, heads, d).permute(0, 2, 1, 3)
    attn = q @ k.transpose(-2, -1) + bias_tab.double()[None]
    if do_shift:
        mask = O.shift_mask(H, W).double().to(attn.device)
        nW = mask.shape[0]
        attn = (attn.view(-1, nW, heads, 48, 48) + mask[None, :, None]).view(-1, heads, 48, 48)
    ow = (attn.softmax(-1) @ v).transpose(1, 2).reshape(-1, 48, C)
    ref = O.window_reverse(ow.reshape(-1, 3, 4, 4, C), clips, 3, H, W)
    ref = torch.roll(ref, (sy, sx), (2, 3))
    return ref.reshape(-1, C)


def window2d_bias(heads, seed):
    from pgtformer_b200.weights import relative_position_index
    table = randn((245, heads), seed, BIAS_STD).float()
    return table[relative_position_index().view(-1)].view(48, 48, heads).permute(2, 0, 1).contiguous()


WIN2D_SHAPES = [(256, 16, 16, 1), (512, 8, 8, 2)]          # d = 32 / 64 at 8 heads


@pytest.mark.parametrize('C,H,W,clips', WIN2D_SHAPES)
@pytest.mark.parametrize('shifted', [False, True])
@pytest.mark.parametrize('kernel', ['tc_n32', 'mma_sync'])
def test_window_attention_large_scores(C, H, W, clips, shifted, kernel):
    """The wgmma kernel adds the shift mask as an exact fp32 constant: in its fp16 bias table (ulp 0.125 near -144 in
    the log2 domain) a masked key's weight moved by up to 4.4 %, beyond the bound at these scores."""
    o = ops()
    heads = 8
    T = clips * 3 * H * W
    qkv = window_qkv(T, C, 800 + C)
    bias_tab = window2d_bias(heads, 801 + C)
    qd = qkv.to(DEV)
    ref = window2d_reference(qd, clips, H, W, C, heads, bias_tab.to(DEV), shifted)
    s = qd[:256, :C].double() @ qd[:256, C:2 * C].double().t() / math.sqrt(C // heads)
    assert s.abs().max().item() > 200
    out = torch.full((T, C), float('nan'), dtype=torch.bfloat16, device=DEV)
    if kernel == 'mma_sync':
        o.window_attention(qd, clips, H, W, C, heads, 2 if shifted else 0, bias_tab.to(DEV), out)
    else:
        tab16 = o.window_tables(bias_tab.to(DEV))
        r = o.window_attention_tc(qd, clips, H, W, C, heads, 2 if shifted else 0, tab16, out)
        assert r is not None, 'shape not covered by the wgmma kernel'
    torch.cuda.synchronize()
    check_close(out, ref, 'window attention %s C=%d shifted=%s' % (kernel, C, shifted), rel=4e-3)


# (D, H, W, window, shift) -> N = 48, 98, 125 tokens per window
WIN3D = [((3, 8, 8), (3, 4, 4), (1, 2, 2)), ((2, 14, 14), (2, 7, 7), (1, 3, 3)), ((5, 10, 10), (5, 5, 5), (2, 2, 2))]


@pytest.mark.parametrize('geom', WIN3D, ids=['N48', 'N98', 'N125'])
@pytest.mark.parametrize('hd', [16, 32, 64])
@pytest.mark.parametrize('shifted', [False, True])
def test_window3d_attention_large_scores(geom, hd, shifted):
    from oracle import swin3d_oracle as S
    (D, H, W), window, shift = geom
    if not shifted:
        shift = (0, 0, 0)
    B, heads = 1, 8
    C = heads * hd
    T = B * D * H * W
    qkv = window_qkv(T, C, 900 + hd + D)
    ws, ss = S.window_size_for((D, H, W), window, shift)
    N = ws[0] * ws[1] * ws[2]
    table = randn(((2 * window[0] - 1) * (2 * window[1] - 1) * (2 * window[2] - 1), heads), 901 + hd, BIAS_STD).float()
    bias = table[S.relative_position_index(window)[:N, :N].reshape(-1)].view(N, N, heads).permute(2, 0, 1).contiguous()
    out = torch.full((T, C), float('nan'), dtype=torch.bfloat16, device=DEV)
    ops().window3d_attention(qkv.to(DEV), B, D, H, W, C, heads, window, shift, bias.to(DEV), out)
    torch.cuda.synchronize()
    # fp64 reference: exactly swin3d_oracle.block's geometry (these shapes need no padding)
    x = qkv.double().view(B, D, H, W, 3 * C)
    shifted_ = any(v > 0 for v in ss)
    if shifted_:
        x = torch.roll(x, shifts=(-ss[0], -ss[1], -ss[2]), dims=(1, 2, 3))
    xw = S.partition(x, ws)
    q = xw[..., :C].reshape(-1, N, heads, hd).permute(0, 2, 1, 3) * hd ** -0.5
    k = xw[..., C:2 * C].reshape(-1, N, heads, hd).permute(0, 2, 1, 3)
    v = xw[..., 2 * C:].reshape(-1, N, heads, hd).permute(0, 2, 1, 3)
    attn = q @ k.transpose(-2, -1) + bias.double()[None]
    if shifted_:
        mask = S.shift_mask(D, H, W, ws, ss).double()
        attn = (attn.view(-1, mask.shape[0], heads, N, N) + mask[None, :, None]).view(-1, heads, N, N)
    ow = (attn.softmax(-1) @ v).transpose(1, 2).reshape(-1, N, C)
    ref = S.reverse(ow, ws, B, D, H, W)
    if shifted_:
        ref = torch.roll(ref, shifts=ss, dims=(1, 2, 3))
    assert (q @ k.transpose(-2, -1)).abs().max().item() > 200
    check_close(out, ref.reshape(T, C), 'window3d N=%d d=%d shift=%s' % (N, hd, ss), rel=4e-3)


# ==================================================================================================== C. mean offsets
def pack_conv_weight(w):
    """OIHW -> [Cout, k*k*CinPad] bf16, K index = tap*CinPad + c (see include/pgt_b200.h)."""
    co, ci, kh, kw = w.shape
    cp = (ci + 63) // 64 * 64
    wp = torch.zeros(co, kh * kw, cp)
    wp[:, :, :ci] = w.float().permute(0, 2, 3, 1).reshape(co, kh * kw, ci)
    return wp.reshape(co, kh * kw * cp).to(torch.bfloat16).contiguous()


def offset_rows(shape, ratio, seed, sigma=1.0):
    """mu + sigma * n in fp64 with mu / sigma = ratio (mu = sigma * ratio; sigma when ratio = 0)."""
    return ratio * sigma + sigma * randn(shape, seed)


def constant_value(ratio, sigma=1.0):
    return ratio * sigma + 0.75 * sigma


def affine(C, seed):
    return (1 + 0.1 * randn((C,), seed)).float(), (0.1 * randn((C,), seed + 1)).float()


def ln64(x, g, b, eps=1e-5):
    x = x.double()
    m = x.mean(-1, keepdim=True)
    var = ((x - m) ** 2).mean(-1, keepdim=True)
    y = (x - m) / torch.sqrt(var + eps)
    return y * g.double() + b.double() if g is not None else y


LN_CASES = [(dt, r) for dt in ('f32',) for r in RATIOS_F32] + [(dt, r) for dt in ('bf16',) for r in RATIOS_BF16]


@pytest.mark.parametrize('dt,ratio', LN_CASES)
@pytest.mark.parametrize('C', [256, 512])
@pytest.mark.parametrize('with_pos', [False, True])
def test_layernorm_mean_offset(dt, ratio, C, with_pos):
    o = ops()
    T = 1000
    x = offset_rows((T, C), ratio, 1000 + C + ratio)
    x[0] = constant_value(ratio)
    x = x.to(torch.float32 if dt == 'f32' else torch.bfloat16).to(DEV)
    g, b = affine(C, 1001)
    g, b = g.to(DEV), b.to(DEV)
    y = torch.full((T, C), float('nan'), dtype=torch.bfloat16, device=DEV)
    pos = y2 = None
    if with_pos:
        pos = randn((T, C), 1003).to(torch.bfloat16).to(DEV)
        y2 = torch.full_like(y, float('nan'))
    o.layernorm(x, g, b, y, pos=pos, out2=y2)
    torch.cuda.synchronize()
    ref = ln64(x, g, b)
    what = 'layernorm %s C=%d mu/sigma=%d' % (dt, C, ratio)
    check_close(y, ref, what)
    if with_pos:
        check_close(y2, ref + pos.double(), what + ' + pos')


@pytest.mark.parametrize('dt,ratio', LN_CASES)
@pytest.mark.parametrize('C', [256, 512])
def test_layernorm_constant_row(dt, ratio, C):
    """A constant row (sigma = 0) at mean mu: its output is beta, to one bf16 ulp + 1e-3 * max|beta|."""
    o = ops()
    T = 64
    x = torch.full((T, C), constant_value(ratio), dtype=torch.float64)
    x = x.to(torch.float32 if dt == 'f32' else torch.bfloat16).to(DEV)
    g, b = affine(C, 1001)
    y = torch.full((T, C), float('nan'), dtype=torch.bfloat16, device=DEV)
    o.layernorm(x, g.to(DEV), b.to(DEV), y)
    torch.cuda.synchronize()
    check_close(y, b[None].expand(T, C), 'layernorm %s C=%d constant row at mu = %g' % (dt, C, constant_value(ratio)))


@pytest.mark.parametrize('ratio', RATIOS_BF16)
@pytest.mark.parametrize('folded', [False, True])
def test_ln_linear_mean_offset(ratio, folded):
    o = ops()
    T, C, N = 1000, 256, 512
    x = offset_rows((T, C), ratio, 1100 + ratio)
    x[0] = constant_value(ratio)
    x = x.to(torch.bfloat16).to(DEV)
    g, b = affine(C, 1101)
    w, wb = randn((N, C), 1103, C ** -0.5), randn((N,), 1104, 0.1)
    g, b, w, wb = g.double().to(DEV), b.double().to(DEV), w.to(DEV), wb.to(DEV)
    out = torch.full((T, N), float('nan'), dtype=torch.bfloat16, device=DEV)
    what = 'LN + linear mu/sigma=%d%s' % (ratio, ' folded' if folded else '')
    if folded:
        o.ln_linear(x, None, None, (w * g[None]).to(torch.bfloat16), (wb + w @ b).float(), out)
        ref = ln64(x, g, b) @ w.t() + wb
        rel = 4e-3
    else:
        wq = w.to(torch.bfloat16)
        o.ln_linear(x, g.float(), b.float(), wq, wb.float(), out)
        ref = ln64(x, g, b).to(torch.bfloat16).double() @ wq.double().t() + wb      # LN(x) is a bf16 MMA operand
        rel = 3e-3
    torch.cuda.synchronize()
    check_close(out, ref, what, rel=rel)


@pytest.mark.parametrize('ratio', RATIOS_BF16)
@pytest.mark.parametrize('folded', [False, True])
def test_swin_mlp_mean_offset(ratio, folded):
    """sigma = 1/4, so that the residual x stays comparable to the MLP branch at the largest offset."""
    o = ops()
    T, C, sig = 1000, 256, 0.25
    x = offset_rows((T, C), ratio, 1200 + ratio, sig)
    x[0] = constant_value(ratio, sig)
    x = x.to(torch.bfloat16).to(DEV)
    g, b = affine(C, 1201)
    w1, b1 = randn((C, C), 1203, C ** -0.5).to(DEV), randn((C,), 1204, 0.1).to(DEV)
    w2, b2 = randn((C, C), 1205, C ** -0.5).to(torch.bfloat16).to(DEV), randn((C,), 1206, 0.1).to(DEV)
    g, b = g.double().to(DEV), b.double().to(DEV)
    out = torch.full((T, C), float('nan'), dtype=torch.bfloat16, device=DEV)
    if folded:
        o.swin_mlp(x, None, None, (w1 * g[None]).to(torch.bfloat16), (b1 + w1 @ b).float(), w2, b2.float(), out)
        hdn = F.gelu(ln64(x, g, b) @ w1.t() + b1)
        rel = 6e-3
    else:
        w1q = w1.to(torch.bfloat16)
        o.swin_mlp(x, g.float(), b.float(), w1q, b1.float(), w2, b2.float(), out)
        y = ln64(x, g, b).to(torch.bfloat16).double()                                # bf16 MMA operands
        hdn = F.gelu(y @ w1q.double().t() + b1).to(torch.bfloat16).double()
        rel = 4e-3
    torch.cuda.synchronize()
    ref = x.double() + hdn @ w2.double().t() + b2
    check_close(out, ref, 'swin mlp mu/sigma=%d%s' % (ratio, ' folded' if folded else ''), rel=rel)


def gn64(x, g, b, eps=1e-6, stats_of=None):
    """fp64 GroupNorm(32) of channels-last x [F, P, C]; statistics of `stats_of` (default x itself)."""
    Fr, P, C = x.shape
    s = (x if stats_of is None else stats_of).double().reshape(Fr, P, 32, C // 32)
    m = s.mean((1, 3), keepdim=True)
    var = ((s - m) ** 2).mean((1, 3), keepdim=True)
    y = (x.double().reshape(Fr, P, 32, C // 32) - m) / torch.sqrt(var + eps)
    return y.reshape(Fr, P, C) * g.double() + b.double()


def offset_groups(Fr, P, C, ratio, seed):
    """mu + n; group 3 of frame 0 exactly constant."""
    x = offset_rows((Fr, P, C), ratio, seed)
    x[0, :, 3 * (C // 32):4 * (C // 32)] = constant_value(ratio)
    return x


@pytest.mark.parametrize('ratio', RATIOS_BF16)
@pytest.mark.parametrize('C', [256, 512])
def test_groupnorm_silu_mean_offset(ratio, C):
    _groupnorm_offset(ratio, C, False)


# y = x * a + b with a = gamma / sqrt(var + eps), b = beta - mean * a: for a constant group (var = 0, a ~ 1e3 gamma)
# at an offset, x * a and b cancel, and the rounding of b (|mean * a| ~ 6e4 at mean 64) leaves up to ~2e-3 on beta.
# The whole-tensor bound above holds; beta itself to one ulp + 1e-3 * max|beta| does not.  Not changed here: the
# fix ((x - mean) * a + beta) changes the bits of every GroupNorm of the codec.
GN_CONST_XFAIL = pytest.mark.xfail(strict=True, reason='gn_apply: x * a + b cancels for a constant group at an offset')


@pytest.mark.parametrize('ratio,C', [(0, 256), (0, 512), (8, 512),
                                     pytest.param(8, 256, marks=GN_CONST_XFAIL),
                                     pytest.param(64, 256, marks=GN_CONST_XFAIL),
                                     pytest.param(64, 512, marks=GN_CONST_XFAIL)])
def test_groupnorm_silu_constant_group(ratio, C):
    _groupnorm_offset(ratio, C, True)


def _groupnorm_offset(ratio, C, constant_group_only):
    o = ops()
    Fr, HW = 2, 1024
    x = offset_groups(Fr, HW, C, ratio, 1300 + C + ratio).to(torch.bfloat16).to(DEV)
    g, b = affine(C, 1301)
    g, b = g.to(DEV), b.to(DEV)
    out = torch.full((Fr, HW, C), float('nan'), dtype=torch.bfloat16, device=DEV)
    cpg = C // 32
    for silu in (True, False):
        o.groupnorm_silu(x, g, b, out, silu=silu)
        torch.cuda.synchronize()
        ref = gn64(x, g, b)
        ref = F.silu(ref) if silu else ref
        what = 'groupnorm%s C=%d mu/sigma=%d' % ('+silu' if silu else '', C, ratio)
        if constant_group_only:
            check_close(out[0, :, 3 * cpg:4 * cpg], ref[0, :, 3 * cpg:4 * cpg], what + ': constant group')
        else:
            check_close(out, ref, what)


@pytest.mark.parametrize('ratio', RATIOS_BF16)
@pytest.mark.parametrize('producer', ['linear', 'conv'])
def test_groupnorm_fused_stats_mean_offset(ratio, producer):
    """GroupNorm(32)+SiLU from the (sum, sumsq) a linear / conv epilogue accumulated from its fp32 results.  The offset
    rides on the producer's bias; group 3 gets zero weights, so it is exactly constant.  The reference takes the
    statistics of the fp64 producer output (what the epilogue sums) and applies them to the bf16 tensor the kernel reads."""
    o = ops()
    Fr, H, W, Cin, Cout = 2, 16, 16, 128, 256
    cpg = Cout // 32
    x = randn((Fr, H, W, Cin), 1400).to(torch.bfloat16)
    bias = (ratio + 0.1 * randn((Cout,), 1402)).float()
    bias[3 * cpg:4 * cpg] = constant_value(ratio)
    g, b = affine(Cout, 1403)
    y = torch.empty(Fr, H, W, Cout, dtype=torch.bfloat16, device=DEV)
    if producer == 'linear':
        w = randn((Cout, Cin), 1401, Cin ** -0.5).to(torch.bfloat16)
        w[3 * cpg:4 * cpg] = 0
        tpf = H * W // 128
        stats = torch.zeros(Fr * tpf * 4 * 64, dtype=torch.float32, device=DEV)
        o.linear(x.to(DEV), w.to(DEV), y, bias=bias.to(DEV), gn_stats=stats)
        y64 = x.double() @ w.double().t() + bias.double()
    else:
        w = randn((Cout, Cin, 3, 3), 1401, (9 * Cin) ** -0.5).to(torch.bfloat16)
        w[3 * cpg:4 * cpg] = 0
        tpf = o.conv_tiles_per_frame(H, W, Cout)
        assert tpf > 0
        stats = torch.zeros(Fr * tpf * 4 * 64, dtype=torch.float32, device=DEV)
        o.conv(x.to(DEV), pack_conv_weight(w.float()).to(DEV), Cout, y, bias=bias.to(DEV), gn_stats=stats)
        y64 = F.conv2d(x.double().permute(0, 3, 1, 2), w.double(), bias.double(), padding=1).permute(0, 2, 3, 1)
    out = torch.full_like(y, float('nan'))
    o.groupnorm_apply_stats(y, g.to(DEV), b.to(DEV), out, stats, tpf * 4)
    torch.cuda.synchronize()
    ref = F.silu(gn64(y.view(Fr, H * W, Cout), g.to(DEV), b.to(DEV), stats_of=y64.to(DEV).reshape(Fr, H * W, Cout)))
    check_close(out.view(Fr, H * W, Cout), ref, 'fused-stats groupnorm (%s) mu/sigma=%d' % (producer, ratio), rel=3e-3)


@pytest.mark.parametrize('ratio', RATIOS_BF16)
@pytest.mark.parametrize('silu', [True, False])
def test_conv_out_gn_mean_offset(ratio, silu):
    """groupnorm_ab statistics of an offset input, applied inside conv_out_gn: conv3x3(act(GroupNorm(x))) -> fp32
    NCHW, act = SiLU (the decoder tail) or identity (VQGAN's / CodeFormer's generator tail)."""
    o = ops()
    Fr, H, W, Cin, Cout = 2, 32, 24, 64, 3
    x = offset_groups(Fr, H * W, Cin, ratio, 1500 + ratio).view(Fr, H, W, Cin).to(torch.bfloat16).to(DEV)
    g, b = affine(Cin, 1501)
    w = randn((Cout, Cin, 3, 3), 1503, (9 * Cin) ** -0.5).to(torch.bfloat16)
    bias = randn((Cout,), 1504, 0.1).float().to(DEV)
    ab = torch.empty(Fr * 2 * Cin, dtype=torch.float32, device=DEV)
    o.groupnorm_ab(x, g.to(DEV), b.to(DEV), ab)
    out = torch.full((Fr, Cout, H, W), float('nan'), dtype=torch.float32, device=DEV)
    assert o.conv_out_gn(x, ab, pack_conv_weight(w.float()).to(DEV), Cout, bias, out, silu=silu) is not None
    torch.cuda.synchronize()
    act = gn64(x.view(Fr, H * W, Cin), g.to(DEV), b.to(DEV))
    act = (F.silu(act) if silu else act).view(Fr, H, W, Cin)
    act = act.to(torch.bfloat16).double()                                              # the bf16 MMA operand
    ref = F.conv2d(act.permute(0, 3, 1, 2), w.double().to(DEV), bias.double(), padding=1)
    check_close(out, ref, 'conv_out_gn%s mu/sigma=%d' % ('+silu' if silu else '', ratio), rel=4e-3)


ADAIN_CASES = [('f32', r) for r in RATIOS_F32] + [('bf16', r) for r in RATIOS_BF16]


@pytest.mark.parametrize('dt,ratio', ADAIN_CASES)
@pytest.mark.parametrize('HW', [256, 1024])
def test_adain_mean_offset(dt, ratio, HW):
    """Offsets in the content (fp32 or bf16) and the style (bf16, at most 64) inputs; channel 5 of the content and
    channel 7 of the style exactly constant; unbiased variance + eps as in the reference."""
    o = ops()
    Fr, C = 2, 512
    q = offset_rows((Fr, HW, C), ratio, 1600 + ratio + HW)
    q[:, :, 5] = constant_value(ratio)
    sr = min(ratio, 64)
    s = offset_rows((Fr, HW, C), sr, 1601 + ratio + HW, 0.5)
    s[:, :, 7] = constant_value(sr, 0.5)
    q = q.to(torch.float32 if dt == 'f32' else torch.bfloat16).to(DEV)
    s = s.to(torch.bfloat16).to(DEV)
    out = torch.full((Fr, HW, C), float('nan'), dtype=torch.bfloat16, device=DEV)
    o.adain(q, s, out)
    torch.cuda.synchronize()
    qd, sd = q.double(), s.double()
    eps = 1e-5
    qm, qs = qd.mean(1, keepdim=True), torch.sqrt(qd.var(1, keepdim=True) + eps)
    sm, ss = sd.mean(1, keepdim=True), torch.sqrt(sd.var(1, keepdim=True) + eps)
    ref = (qd - qm) / qs * ss + sm
    check_close(out, ref, 'adain %s content mu/sigma=%d, style %d' % (dt, ratio, sr))
