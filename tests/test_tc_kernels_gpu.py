"""GPU parity of the round-2 wgmma kernels THROUGH THE C ABI against the CPU oracle:
  * pgt_window_attention_tc (TMA + wgmma shifted-window attention core) vs the oracle's roll / window_partition /
    attention / window_reverse, every box layout (interior, x-wrapped, y-wrapped, corner), both P V operand modes;
  * pgt_l2_argmin_tc (tensor-core scores + certified window + exact re-evaluation) vs an fp64 argmin — bit-exact in the
    four SURVEY section-7 regimes, at small T (direct fp64 differences) and at the BASELINE sizes T = 49152 / 98304.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def ops():
    from pgtformer_b200 import ops as o
    return o


def rnd(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g) * scale


def window_reference(qkv, clips, H, W, C, heads, bias_tab, shifted):
    from oracle import pgt_oracle as O
    d = C // heads
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
    return ref.reshape(-1, C)


@pytest.mark.parametrize('C,H,W,clips', [(256, 16, 16, 1), (512, 8, 8, 2), (256, 32, 32, 1), (512, 4, 4, 1), (512, 4, 4, 3),
                                         (256, 8, 16, 1), (256, 12, 8, 1)])
@pytest.mark.parametrize('shifted', [False, True])
@pytest.mark.parametrize('mode_n64', [0, 1])
def test_window_attention_tc(C, H, W, clips, shifted, mode_n64):
    """Core only (q / kv / proj identity).  P is rounded to bf16 before P V (as in every flash-style kernel), which
    is the 4e-3 * max|ref| term on top of the one-ulp bound of the bf16 output."""
    from pgtformer_b200.weights import relative_position_index
    o = ops()
    heads = 8
    T = clips * 3 * H * W
    qkv = rnd((T, 3 * C), 100, 1.0).bfloat16()
    table = 0.5 * rnd((245, heads), 101)
    idx = relative_position_index()
    bias_tab = table[idx.view(-1)].view(48, 48, heads).permute(2, 0, 1).contiguous()
    tab16 = o.window_tables(bias_tab.to(DEV))
    out = torch.full((T, C), float('nan'), dtype=torch.bfloat16, device=DEV)
    r = o.window_attention_tc(qkv.to(DEV), clips, H, W, C, heads, 2 if shifted else 0, tab16, out, mode_n64=mode_n64)
    assert r is not None, 'shape not covered by the wgmma kernel'
    torch.cuda.synchronize()
    ref = window_reference(qkv, clips, H, W, C, heads, bias_tab, shifted)
    got = out.float().cpu()
    assert torch.isfinite(got).all(), 'non-finite / unwritten output rows'
    err = (got - ref).abs()
    tol = ref.abs() * 2.0 ** -8 + 4e-3 * ref.abs().max()
    assert not (err > tol).any(), 'max err %.3e (max|ref| %.3e), %d bad' % (err.max(), ref.abs().max(), int((err > tol).sum()))


def test_window_attention_tc_matches_mma_sync_kernel():
    """The round-1 mma.sync kernel and the wgmma kernel agree to bf16 rounding on a batch large enough that every
    CTA of the persistent grid processes several window pairs."""
    from pgtformer_b200.weights import relative_position_index
    o = ops()
    C, H, W, clips, heads = 256, 64, 64, 3, 8
    T = clips * 3 * H * W
    qkv = rnd((T, 3 * C), 7, 1.0).bfloat16().to(DEV)
    table = 0.5 * rnd((245, heads), 8)
    bias_tab = table[relative_position_index().view(-1)].view(48, 48, heads).permute(2, 0, 1).contiguous().to(DEV)
    tab16 = o.window_tables(bias_tab)
    for shift in (0, 2):
        a = torch.empty(T, C, dtype=torch.bfloat16, device=DEV)
        b = torch.empty(T, C, dtype=torch.bfloat16, device=DEV)
        o.window_attention(qkv, clips, H, W, C, heads, shift, bias_tab, a)
        assert o.window_attention_tc(qkv, clips, H, W, C, heads, shift, tab16, b) is not None
        d = (a.float() - b.float()).abs().max().item()
        assert d <= 4e-3 * a.float().abs().max().item() + 2.0 ** -7, d


# ------------------------------------------------------------------------------------ L2 argmin
def exact_argmin_small(cb, z):
    from oracle import pgt_oracle as O
    return O.l2_argmin_exact(cb, z)[0]


def make_regime(regime, T, seed, cb):
    """The four regimes of SURVEY section 7 (bit-exact argmin study)."""
    if regime == 'random':                       # small margins everywhere
        return rnd((T, 512), seed), cb
    if regime == 'random_scaled':                # z and codebook at very different scales
        return 30.0 * rnd((T, 512), seed), cb
    if regime == 'near_code':                    # trained-like: z = code + noise
        pick = torch.randint(0, 1024, (T,), generator=torch.Generator().manual_seed(seed + 1))
        return cb[pick] + 0.05 * rnd((T, 512), seed + 2), cb
    cb = cb.clone()                              # duplicated codes: exact ties, lowest index must win
    cb[700] = cb[3]
    cb[701] = cb[3]
    cb[900] = cb[17]
    z = 0.01 * rnd((T, 512), seed + 3)
    z[0::2] += cb[3]
    z[1::2] += cb[17]
    return z, cb


def run_tc(z, cb):
    o = ops()
    T = z.shape[0]
    cbd = cb.to(DEV).contiguous()
    pack = o.codebook_pack(cbd, 1024)
    idx = torch.full((T,), -7, dtype=torch.int64, device=DEV)
    quant = torch.empty(T, 512, dtype=torch.float32, device=DEV)
    o.l2_argmin_tc(z.to(DEV).contiguous(), cbd, pack, 1024, idx, quant)
    torch.cuda.synchronize()
    return idx.cpu(), quant.cpu()


@pytest.mark.parametrize('regime', ['random', 'random_scaled', 'near_code', 'duplicates'])
@pytest.mark.parametrize('T', [775, 128, 1])
def test_l2_argmin_tc_bit_exact_small(synth_sd, regime, T):
    cb0 = synth_sd['quantizer.codebooks.0.weight'].clone()
    z, cb = make_regime(regime, T, 90, cb0)
    idx, quant = run_tc(z, cb)
    ref = exact_argmin_small(cb, z)                 # the oracle drops the padding row itself
    assert torch.equal(idx, ref), 'mismatches: %d of %d' % (int((idx != ref).sum()), T)
    assert torch.equal(quant, cb[ref])
    if regime == 'duplicates':
        assert set(idx.tolist()) <= {3, 17}


def test_l2_argmin_tc_degenerate_codebooks():
    """All-equal and all-zero codebooks: every code is inside the certificate window, so every token takes the
    exhaustive path; the answer is still the first index."""
    z = rnd((300, 512), 5)
    for cb in (torch.zeros(1025, 512), rnd((1, 512), 6).expand(1025, 512).contiguous()):
        idx, _ = run_tc(z, cb)
        assert (idx == 0).all()


def fp64_argmin_big(cb, z, chunk=4096):
    """fp64 argmin of ||z - e||^2 at BASELINE sizes: matmul form in fp64 (error ~1e-15 relative), direct fp64 differences
    wherever the top-2 margin of the matmul form is below 1e-9 relative."""
    cb64 = cb.double()
    n2 = (cb64 * cb64).sum(1)
    out = torch.empty(z.shape[0], dtype=torch.int64)
    for s in range(0, z.shape[0], chunk):
        zz = z[s:s + chunk].double()
        d = n2[None] - 2.0 * zz @ cb64.t()
        top = d.topk(2, dim=1, largest=False)
        idx = top.indices[:, 0].clone()
        z2 = (zz * zz).sum(1)
        close = (top.values[:, 1] - top.values[:, 0]) <= 1e-9 * (top.values[:, 0] + z2).abs()
        for t in close.nonzero().flatten().tolist():
            dd = ((zz[t][None] - cb64) ** 2).sum(1)
            idx[t] = int(dd.argmin())
        out[s:s + chunk] = idx
    return out


@pytest.mark.parametrize('T', [49152, 98304])
@pytest.mark.parametrize('regime', ['random', 'random_scaled', 'near_code', 'duplicates'])
def test_l2_argmin_tc_bit_exact_baseline_sizes(synth_sd, regime, T):
    """T = 49152 is BASELINE configs[2] (16 clips of 512^2), 98304 is configs[4] (8 clips of 1024^2)."""
    cb0 = synth_sd['quantizer.codebooks.0.weight'].clone()
    z, cb = make_regime(regime, T, 123, cb0)
    idx, quant = run_tc(z, cb)
    if regime == 'duplicates':
        # exact ties: the matmul form cannot order them; the answer is known by construction (z sits on code 3 / 17)
        ref = torch.full((T,), 3, dtype=torch.int64)
        ref[1::2] = 17
    else:
        ref = fp64_argmin_big(cb[:1024], z)
    bad = int((idx != ref).sum())
    assert bad == 0, '%d mismatches vs the fp64 argmin at T = %d (%s)' % (bad, T, regime)
    assert torch.equal(quant[::97], cb[ref[::97]])


@pytest.mark.parametrize('K,E,T', [(768, 512, 40000), (512, 256, 33333), (256, 128, 700), (1024, 384, 20001)])
def test_l2_argmin_tc_other_codebook_shapes(synth_sd, K, E, T):
    """Pair sweep with an odd number of N-tiles (the accumulator buffers alternate across tiles), fewer k-blocks, several
    several 128-token tiles per CTA and a ragged last tile."""
    o = ops()
    cb = synth_sd['quantizer.codebooks.0.weight'][:K, :E].contiguous()
    z = rnd((T, E), 31 + K)
    cbd = cb.to(DEV)
    idx = torch.full((T,), -7, dtype=torch.int64, device=DEV)
    quant = torch.empty(T, E, dtype=torch.float32, device=DEV)
    o.l2_argmin_tc(z.to(DEV), cbd, o.codebook_pack(cbd, K), K, idx, quant)
    torch.cuda.synchronize()
    ref = fp64_argmin_big(cb, z)
    bad = int((idx.cpu() != ref).sum())
    assert bad == 0, '%d mismatches vs the fp64 argmin (K=%d E=%d T=%d)' % (bad, K, E, T)
    assert torch.equal(quant.cpu()[::53], cb[ref[::53]])


def test_l2_argmin_tc_equals_exhaustive_kernel(synth_sd):
    o = ops()
    cb = synth_sd['quantizer.codebooks.0.weight'].to(DEV).contiguous()
    z = rnd((5000, 512), 77).to(DEV)
    a = torch.empty(5000, dtype=torch.int64, device=DEV)
    b = torch.empty(5000, dtype=torch.int64, device=DEV)
    o.l2_argmin(z, cb, 1024, a)
    o.l2_argmin_tc(z, cb, o.codebook_pack(cb, 1024), 1024, b)
    assert torch.equal(a, b)


# ------------------------------------------------------------------------------------ decoder tail
@pytest.mark.parametrize('F,H,W', [(3, 32, 32), (2, 64, 48), (1, 16, 8)])
def test_conv_out_gn_fused(F, H, W):
    """norm_out -> SiLU -> conv_out (64 -> 3) as one kernel vs the oracle ops on the same bf16-rounded input / weights.
    The kernel rounds the activated tensor to bf16 (MMA operand), as the separate GroupNorm pass did; the oracle side
    emulates that rounding, so what remains is the approximate SiLU flipping an occasional bf16 ulp (3e-3 * max|ref|)."""
    import torch.nn.functional as Fn
    o = ops()
    x = rnd((F, H, W, 64), 31, 1.5).bfloat16()
    gamma, beta = 1.0 + 0.2 * rnd((64,), 32), 0.1 * rnd((64,), 33)
    w = (0.05 * rnd((3, 64, 3, 3), 34))
    bias = 0.1 * rnd((3,), 35)
    wp = w.permute(0, 2, 3, 1).reshape(3, 9 * 64).bfloat16().contiguous()
    xd = x.to(DEV)
    ab = o.groupnorm_ab(xd, gamma.to(DEV), beta.to(DEV), torch.empty(F * 2 * 64, dtype=torch.float32, device=DEV))
    out = torch.full((F, 3, H, W), float('nan'), dtype=torch.float32, device=DEV)
    assert o.conv_out_gn(xd, ab, wp.to(DEV), 3, bias.to(DEV), out) is not None
    torch.cuda.synchronize()
    xn = Fn.group_norm(x.float().permute(0, 3, 1, 2), 32, gamma, beta, eps=1e-6)
    act = (xn * torch.sigmoid(xn)).bfloat16().float()
    ref = Fn.conv2d(act, w.bfloat16().float(), bias, padding=1)
    got = out.cpu()
    assert torch.isfinite(got).all()
    err = (got - ref).abs().max().item()
    assert err <= 3e-3 * ref.abs().max().item(), (err, ref.abs().max().item())


# ------------------------------------------------------------------------------------ TORCH_LIBRARY binding
def test_torch_ops_binding_equals_ctypes_binding(synth_sd):
    """torch.ops.pgt.* and the ctypes binding call the same C entry points: identical bits."""
    from pgtformer_b200 import torch_ops
    from pgtformer_b200.weights import relative_position_index
    o = ops()
    t = torch_ops.load()
    # window attention
    C, H, W, clips, heads = 256, 16, 16, 2, 8
    T = clips * 3 * H * W
    qkv = rnd((T, 3 * C), 1).bfloat16().to(DEV)
    bias = (0.5 * rnd((245, heads), 2))[relative_position_index().view(-1)].view(48, 48, heads).permute(2, 0, 1).contiguous().to(DEV)
    tab = o.window_tables(bias)
    a = torch.empty(T, C, dtype=torch.bfloat16, device=DEV)
    b = torch.empty_like(a)
    o.window_attention_tc(qkv, clips, H, W, C, heads, 2, tab, a)
    t.window_attention(qkv, clips, H, W, C, heads, 2, tab, b)
    assert torch.equal(a, b)
    # codebook kernels
    cb = synth_sd['quantizer.codebooks.0.weight'].to(DEV).contiguous()
    z = rnd((1000, 512), 3).to(DEV)
    i1 = torch.empty(1000, dtype=torch.int64, device=DEV)
    i2 = torch.empty_like(i1)
    o.l2_argmin_tc(z, cb, o.codebook_pack(cb, 1024), 1024, i1)
    cb16, norm = t.codebook_pack(cb, 1024)
    t.l2_argmin(z, cb, cb16, norm, 1024, i2, None)
    assert torch.equal(i1, i2)
    logits = rnd((1000, 1024), 4).to(DEV)
    q1, q2 = torch.empty(1000, 512, device=DEV), torch.empty(1000, 512, device=DEV)
    o.argmax_gather(logits, cb, i1, q1)
    t.argmax_gather(logits, cb, i2, q2)
    assert torch.equal(i1, i2) and torch.equal(q1, q2)
    # GEMM with bias + GELU + residual, flash attention
    x = rnd((300, 192), 5).bfloat16().to(DEV)
    w = rnd((96, 192), 6, 0.1).bfloat16().to(DEV)
    bia = rnd((96,), 7).to(DEV)
    res = rnd((300, 96), 8).bfloat16().to(DEV)
    y1 = torch.empty(300, 96, dtype=torch.bfloat16, device=DEV)
    y2 = torch.empty_like(y1)
    o.linear(x, w, y1, bias=bia, act=o.ACT_GELU, residual=res)
    t.linear(x, w, bia, o.ACT_GELU, res, y2)
    assert torch.equal(y1, y2)
    L = 256
    q, k, v = (rnd((2 * L, 512), 9 + i).bfloat16().to(DEV) for i in range(3))
    m1 = torch.empty(2 * L, 512, dtype=torch.bfloat16, device=DEV)
    m2 = torch.empty_like(m1)
    o.mha(q, k, v, 2, L, 8, 64, m1)
    t.mha_fwd(q, k, v, 2, L, 8, 64, m2)
    assert torch.equal(m1, m2)
