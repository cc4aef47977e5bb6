"""TEST INFRASTRUCTURE ONLY — CPU restatement (PyTorch fp32/fp64, functional, state-dict driven)
of the reference algorithm for the PGTFormer forward path.  It is the *checker*: only tests/,
`__graft_entry__.smoke()` and bench.py's cpu_baseline / `--impl reference` legs may import it.
The product path (pgtformer_b200/, archs/) never does and fails loudly without its CUDA library.

Pinning: the reference ships no golden vectors or tests (SURVEY 4, 8c).  This restatement is
pinned instead against the reference itself (oracle/reference_loader.py imports a reference
checkout): tests/golden/* hold outputs *of the reference* (minted by oracle/make_golden.py: 64x64
in full, 128x128, 512x512 — its unpatched native size — and 1024x1024 as bounded samples) that
tests/test_oracle.py checks this file against.

Every function cites the reference lines it restates.  Unlike the reference it is size-general
(H, W multiples of 64) and batch-general (b clips of 3 frames); SURVEY F4/F5 explain why the
unmodified reference is neither, and reference_loader.generalise_size is the matching patch.
"""
import math

import torch
import torch.nn.functional as F

WIN = (4, 4)
SHIFT = (2, 2)
FRAMES = 3


# --------------------------------------------------------------------------- primitives
def conv(sd, p, x, stride=1, padding=0):
    return F.conv2d(x, sd[p + '.weight'], sd.get(p + '.bias'), stride=stride, padding=padding)


def linear(sd, p, x):
    return F.linear(x, sd[p + '.weight'], sd.get(p + '.bias'))


def group_norm(sd, p, x):
    """Normalize(): GroupNorm(32, eps=1e-6)  (`modules/rstt_layers.py:754-755`)."""
    return F.group_norm(x, 32, sd[p + '.weight'], sd[p + '.bias'], eps=1e-6)


def layer_norm(sd, p, x):
    return F.layer_norm(x, (x.shape[-1],), sd[p + '.weight'], sd[p + '.bias'], eps=1e-5)


def batch_norm_eval(sd, p, x):
    return F.batch_norm(x, sd[p + '.running_mean'], sd[p + '.running_var'], sd[p + '.weight'],
                        sd[p + '.bias'], training=False, eps=1e-5)


def silu(x):
    return x * torch.sigmoid(x)


# --------------------------------------------------------------------------- ResNet blocks
def td_resblock(sd, p, x):
    """TDResnetBlock._forward on 4-D [b*3,C,H,W] (`modules/rstt_layers.py:875-904`):
    GN -> SiLU -> conv3x3 -> GN -> SiLU -> conv3x3 (+ 1x1 nin_shortcut) + x."""
    h = conv(sd, p + '.conv1', silu(group_norm(sd, p + '.norm1', x)), padding=1)
    h = conv(sd, p + '.conv2', silu(group_norm(sd, p + '.norm2', h)), padding=1)
    if (p + '.nin_shortcut.weight') in sd:
        x = conv(sd, p + '.nin_shortcut', x)
    return x + h


def downsample(sd, p, x):
    """pad(0,1,0,1) + conv3x3 stride 2 (`archs/tdcrqvae3_arch.py:67-76`)."""
    return conv(sd, p + '.conv', F.pad(x, (0, 1, 0, 1)), stride=2)


def upsample(sd, p, x):
    """nearest x2 + conv3x3 (`archs/tdcrqvae3_arch.py:45-52`)."""
    return conv(sd, p + '.conv', F.interpolate(x, scale_factor=2.0, mode='nearest'), padding=1)


# --------------------------------------------------------------------------- window attention
def shift_mask(Hp, Wp, dtype=torch.float32):
    """(nW,48,48) mask of {0,-100}: 3x3 region labels of the rolled map, window-partitioned
    (`modules/rstt_layers.py:552-568`)."""
    img = torch.zeros((1, FRAMES, Hp, Wp, 1), dtype=dtype)
    cnt = 0
    for hs in (slice(0, -WIN[0]), slice(-WIN[0], -SHIFT[0]), slice(-SHIFT[0], None)):
        for ws in (slice(0, -WIN[1]), slice(-WIN[1], -SHIFT[1]), slice(-SHIFT[1], None)):
            img[:, :, hs, ws, :] = cnt
            cnt += 1
    mw = window_partition(img).view(-1, FRAMES * WIN[0] * WIN[1])
    am = mw.unsqueeze(1) - mw.unsqueeze(2)
    return torch.where(am != 0, torch.full_like(am, -100.0), torch.zeros_like(am))


def window_partition(x):
    """(B,D,H,W,C) -> (B*nW, D, 4, 4, C)  (`modules/rstt_layers.py:55-70`)."""
    B, D, H, W, C = x.shape
    x = x.view(B, D, H // WIN[0], WIN[0], W // WIN[1], WIN[1], C)
    return x.permute(0, 2, 4, 1, 3, 5, 6).contiguous().view(-1, D, WIN[0], WIN[1], C)


def window_reverse(win, B, D, H, W):
    """(`modules/rstt_layers.py:72-88`)."""
    x = win.view(B, H // WIN[0], W // WIN[1], D, WIN[0], WIN[1], -1)
    return x.permute(0, 3, 1, 4, 2, 5, 6).contiguous().view(B, D, H, W, -1)


def window_attention(sd, p, xw, heads, mask=None):
    """WindowAttention3D.forward (`modules/rstt_layers.py:195-234`): q scaled by d^-1/2,
    + relative-position bias (245x8 table via the 48x48 index), + {0,-100} shift mask, softmax."""
    B_, N, C = xw.shape
    d = C // heads
    q = linear(sd, p + '.q', xw).view(B_, N, heads, d).permute(0, 2, 1, 3) * (d ** -0.5)
    kv = linear(sd, p + '.kv', xw).view(B_, N, 2, heads, d).permute(2, 0, 3, 1, 4)
    k, v = kv[0], kv[1]
    attn = q @ k.transpose(-2, -1)
    idx = sd[p + '.relative_position_index'].view(-1)
    bias = sd[p + '.relative_position_bias_table'][idx].view(N, N, heads).permute(2, 0, 1)
    attn = attn + bias.unsqueeze(0)
    if mask is not None:
        nW = mask.shape[0]
        attn = (attn.view(B_ // nW, nW, heads, N, N) + mask.to(attn.dtype)[None, :, None]).view(-1, heads, N, N)
    attn = attn.softmax(-1)
    out = (attn @ v).transpose(1, 2).reshape(B_, N, C)
    return linear(sd, p + '.proj', out)


def swin_block(sd, p, x, heads, shifted, mask):
    """VSTSREncoderTransformerBlock.forward on (B,D,H,W,C) (`modules/rstt_layers.py:284-338`);
    H, W are multiples of 4 on this path so the pad branch is a no-op."""
    B, D, H, W, C = x.shape
    assert H % WIN[0] == 0 and W % WIN[1] == 0
    do_shift = shifted and H > WIN[0] and W > WIN[1]       # get_window_size (:90-114)
    h = layer_norm(sd, p + '.norm1', x)
    if do_shift:
        h = torch.roll(h, shifts=(-SHIFT[0], -SHIFT[1]), dims=(2, 3))
    xw = window_partition(h).view(-1, D * WIN[0] * WIN[1], C)
    aw = window_attention(sd, p + '.attn', xw, heads, mask if do_shift else None)
    h = window_reverse(aw.view(-1, D, WIN[0], WIN[1], C), B, D, H, W)
    if do_shift:
        h = torch.roll(h, shifts=SHIFT, dims=(2, 3))
    x = x + h
    m = linear(sd, p + '.mlp.fc1', layer_norm(sd, p + '.norm2', x))
    m = linear(sd, p + '.mlp.fc2', F.gelu(m))                # exact-erf GELU (:116-132)
    return x + m


def encoder_layer(sd, p, x4, heads, depth=2):
    """EncoderLayer.forward (`modules/rstt_layers.py:535-575`); x4 is [b*3,C,H,W]."""
    BD, C, H, W = x4.shape
    x = x4.view(BD // FRAMES, FRAMES, C, H, W).permute(0, 1, 3, 4, 2)
    mask = shift_mask(H, W, x4.dtype) if (H > WIN[0] and W > WIN[1]) else None
    for i in range(depth):
        x = swin_block(sd, '%s.blocks.%d' % (p, i), x, heads, shifted=(i % 2 == 1), mask=mask)
    return x.permute(0, 1, 4, 2, 3).reshape(BD, C, H, W)


# --------------------------------------------------------------------------- encoder / decoder
def encoder_forward(sd, arch, x):
    """Encoder.forward (`archs/tdcrqvae3_arch.py:540-573`) -> (h [b*3,z,H/16,W/16], per-level feats)."""
    h = conv(sd, 'encoder.conv_in', x, padding=1)
    feats = []
    for lvl in range(arch.num_levels):
        for b in range(arch.num_res_blocks):
            h = td_resblock(sd, 'encoder.down.%d.block.%d' % (lvl, b), h)
            if arch.level_has_attn[lvl]:
                h = encoder_layer(sd, 'encoder.down.%d.attn.%d' % (lvl, b), h, arch.num_heads[lvl], arch.depths[lvl])
        feats.append(h)
        if lvl != arch.num_levels - 1:
            h = downsample(sd, 'encoder.down.%d.downsample' % lvl, h)
    h = td_resblock(sd, 'encoder.mid.block_1', h)
    h = encoder_layer(sd, 'encoder.mid.attn_1', h, arch.num_heads[-1], arch.depths[-1])
    h = td_resblock(sd, 'encoder.mid.block_2', h)
    h = conv(sd, 'encoder.conv_out', silu(group_norm(sd, 'encoder.norm_out', h)), padding=1)
    return h, feats


def decoder_forward(sd, arch, z, enc_feats=None, w=0.0):
    """Decoder.forward (`archs/tdcrqvae3_arch.py:672-707`); with enc_feats and w>0 it is the
    hand-inlined variant of `archs/pgtformer_arch.py:680-710` (SFT fusion after each level)."""
    h = conv(sd, 'decoder.conv_in', z, padding=1)
    h = td_resblock(sd, 'decoder.mid.block_1', h)
    h = encoder_layer(sd, 'decoder.mid.attn_1', h, arch.num_heads[-1], arch.depths[-1])
    h = td_resblock(sd, 'decoder.mid.block_2', h)
    for lvl in reversed(range(arch.num_levels)):
        for b in range(arch.num_res_blocks + 1):
            h = td_resblock(sd, 'decoder.up.%d.block.%d' % (lvl, b), h)
            if arch.level_has_attn[lvl]:
                h = encoder_layer(sd, 'decoder.up.%d.attn.%d' % (lvl, b), h, arch.num_heads[lvl], arch.depths[lvl])
        if enc_feats is not None and lvl in arch.fuse_level_key and w > 0:
            h = fuse_sft(sd, 'fuse_convs_dict.' + arch.fuse_level_key[lvl], enc_feats[lvl], h, w)
        if lvl != 0:
            h = upsample(sd, 'decoder.up.%d.upsample' % lvl, h)
    return conv(sd, 'decoder.conv_out', silu(group_norm(sd, 'decoder.norm_out', h)), padding=1)


def sft_resblock(sd, p, x):
    """ResBlock (`archs/pgtformer_arch.py:409-432`)."""
    h = conv(sd, p + '.conv1', silu(group_norm(sd, p + '.norm1', x)), padding=1)
    h = conv(sd, p + '.conv2', silu(group_norm(sd, p + '.norm2', h)), padding=1)
    if (p + '.conv_out.weight') in sd:
        x = conv(sd, p + '.conv_out', x)
    return h + x


def fuse_sft(sd, p, enc, dec, w):
    """Fuse_sft_block.forward (`archs/pgtformer_arch.py:460-484`); enc, dec are [b*3,C,h,w]."""
    BD, C, h, wf = enc.shape
    b, d = BD // FRAMES, FRAMES
    enct = conv(sd, p + '.tconvenc', enc).contiguous().view(b, d * 32, h, wf)
    dect = conv(sd, p + '.tconvdec', dec).contiguous().view(b, d * 32, h, wf)
    fut = conv(sd, p + '.tfusion0', torch.cat([enct, dect], 1)).contiguous().view(b * d, 32, h, wf)
    fut = conv(sd, p + '.tfusion1', fut)
    e = sft_resblock(sd, p + '.encode_enc', torch.cat([enc, dec, fut], 1))
    scale = conv(sd, p + '.scale.2', F.leaky_relu(conv(sd, p + '.scale.0', e, padding=1), 0.2), padding=1)
    shift = conv(sd, p + '.shift.2', F.leaky_relu(conv(sd, p + '.shift.0', e, padding=1), 0.2), padding=1)
    return dec + w * (dec * scale + shift)


# --------------------------------------------------------------------------- parsing net
def _cbr(sd, p, x, stride=1, padding=1):
    return F.relu(batch_norm_eval(sd, p + '.bn', conv(sd, p + '.conv', x, stride, padding)))


def _basic_block(sd, p, x, stride):
    r = F.relu(batch_norm_eval(sd, p + '.bn1', conv(sd, p + '.conv1', x, stride, 1)))
    r = batch_norm_eval(sd, p + '.bn2', conv(sd, p + '.conv2', r, 1, 1))
    if (p + '.downsample.0.weight') in sd:
        x = batch_norm_eval(sd, p + '.downsample.1', conv(sd, p + '.downsample.0', x, stride))
    return F.relu(x + r)


def _arm(sd, p, x):
    feat = _cbr(sd, p + '.conv', x)
    att = feat.mean(dim=(2, 3), keepdim=True)
    att = torch.sigmoid(batch_norm_eval(sd, p + '.bn_atten', conv(sd, p + '.conv_atten', att)))
    return feat * att


def bisenet(sd, p, x):
    """BiSeNet.forward (`archs/pgtformer_arch.py:365-379`; ResNet18 :91-100, ContextPath :228-249,
    FFM :324-334) -> [b*3,57,H/16,W/16]; heads 1,2 bilinear(align_corners) to H/16."""
    H, W = x.shape[2:]
    r = p + '.cp.resnet'
    t = F.relu(batch_norm_eval(sd, r + '.bn1', conv(sd, r + '.conv1', x, 2, 3)))
    t = F.max_pool2d(t, 3, 2, 1)
    feats = []
    for li, stride in ((1, 1), (2, 2), (3, 2), (4, 2)):
        t = _basic_block(sd, '%s.layer%d.0' % (r, li), t, stride)
        t = _basic_block(sd, '%s.layer%d.1' % (r, li), t, 1)
        feats.append(t)
    feat8, feat16, feat32 = feats[1], feats[2], feats[3]
    avg = _cbr(sd, p + '.cp.conv_avg', feat32.mean(dim=(2, 3), keepdim=True), padding=0)
    f32 = _arm(sd, p + '.cp.arm32', feat32) + avg
    f32 = _cbr(sd, p + '.cp.conv_head32', F.interpolate(f32, feat16.shape[2:], mode='nearest'))
    f16 = _arm(sd, p + '.cp.arm16', feat16) + f32
    f16 = _cbr(sd, p + '.cp.conv_head16', F.interpolate(f16, feat8.shape[2:], mode='nearest'))
    fcat = _cbr(sd, p + '.ffm.convblk', torch.cat([feat8, f16], 1), padding=0)
    att = fcat.mean(dim=(2, 3), keepdim=True)
    att = torch.sigmoid(conv(sd, p + '.ffm.conv2', F.relu(conv(sd, p + '.ffm.conv1', att))))
    fuse = fcat * att + fcat
    o0 = conv(sd, p + '.conv_out.conv_out', _cbr(sd, p + '.conv_out.conv', fuse))
    o1 = conv(sd, p + '.conv_out16.conv_out', _cbr(sd, p + '.conv_out16.conv', f16))
    o2 = conv(sd, p + '.conv_out32.conv_out', _cbr(sd, p + '.conv_out32.conv', f32))
    size = (H // 16, W // 16)
    o0 = F.interpolate(o0, size, mode='bilinear', align_corners=True)
    o1 = F.interpolate(o1, size, mode='bilinear', align_corners=True)
    return torch.cat([o0, o1, o2], 1)


# --------------------------------------------------------------------------- global transformer
def transformer_sa_layer(sd, p, tgt, pos, heads=8):
    """TransformerSALayer.forward (`archs/codeformer_arch.py:121-137`) with nn.MultiheadAttention
    restated: q = k = LN(x)+pos, v = LN(x); tgt, pos are [L, b, E] (sequence first)."""
    L, B, E = tgt.shape
    d = E // heads
    t2 = layer_norm(sd, p + '.norm1', tgt)
    qk_in = t2 + pos
    Wi, bi = sd[p + '.self_attn.in_proj_weight'], sd[p + '.self_attn.in_proj_bias']
    q = F.linear(qk_in, Wi[:E], bi[:E])
    k = F.linear(qk_in, Wi[E:2 * E], bi[E:2 * E])
    v = F.linear(t2, Wi[2 * E:], bi[2 * E:])
    sh = lambda a: a.reshape(L, B * heads, d).transpose(0, 1)      # [B*heads, L, d]
    q, k, v = sh(q), sh(k), sh(v)
    attn = torch.softmax((q * (1.0 / math.sqrt(d))) @ k.transpose(1, 2), dim=-1)
    o = (attn @ v).transpose(0, 1).reshape(L, B, E)
    tgt = tgt + linear(sd, p + '.self_attn.out_proj', o)
    t2 = layer_norm(sd, p + '.norm2', tgt)
    return tgt + linear(sd, p + '.linear2', F.gelu(linear(sd, p + '.linear1', t2)))


# --------------------------------------------------------------------------- codebook ops
def l2_distances(codebook_weight, x):
    """VQEmbedding.compute_distances (`archs/tdcrqvae3_arch.py:99-119`): ||x||^2+||e||^2-2 x.e^T
    over codebook rows [:-1] (padding row excluded)."""
    e_t = codebook_weight[:-1].t()
    xf = x.reshape(-1, e_t.shape[0])
    return torch.addmm(xf.pow(2.).sum(1, keepdim=True) + e_t.pow(2.).sum(0, keepdim=True), xf, e_t,
                       alpha=-2.0).reshape(*x.shape[:-1], -1)


def l2_argmin(codebook_weight, x):
    """find_nearest_embedding (`archs/tdcrqvae3_arch.py:121-126`): first-minimum index."""
    return l2_distances(codebook_weight, x).argmin(dim=-1)


def l2_argmin_exact(codebook_weight, x):
    """fp64 adjudicator: argmin_k ||x - e_k||^2 evaluated directly in float64, lowest index on
    ties.  fp32 addmm summation order is library-defined, so bit-exactness of the CUDA kernel is
    asserted against this (SURVEY 7 'Bit-exact argmin'), with the fp32 formula as a cross-check."""
    e = codebook_weight[:-1].double()
    xf = x.reshape(-1, e.shape[1]).double()
    d = (xf * xf).sum(1, keepdim=True) + (e * e).sum(1)[None] - 2.0 * (xf @ e.t())
    return d.argmin(1).reshape(x.shape[:-1]), d


def embed_code(codebook_weight, codes):
    """RQBottleneck.embed_code for depth 1 (`archs/tdcrqvae3_arch.py:354-368`) -> [...,E] NHWC."""
    return F.embedding(codes[..., 0], codebook_weight)


def adain(content, style, eps=1e-5):
    """adaptive_instance_normalization (`archs/codeformer_arch.py:15-46`): unbiased var + eps."""
    def ms(f):
        b, c = f.shape[:2]
        var = f.reshape(b, c, -1).var(dim=2) + eps
        return f.reshape(b, c, -1).mean(dim=2).view(b, c, 1, 1), var.sqrt().view(b, c, 1, 1)
    sm, ss = ms(style)
    cm, cs = ms(content)
    return (content - cm) / cs * ss + sm


# --------------------------------------------------------------------------- full forwards
IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)


def pgtformer_forward(sd, arch, x, w=1.0, adain_on=True, code_only=False, force_codes=None,
                      return_intermediates=False):
    """PGTFormer.forward (`archs/pgtformer_arch.py:598-714`).  x: [b*3,3,H,W] in [0,1].
    Returns (out, logits [b*3,h,w,1,K], lq_feat NHWC).  `force_codes` teacher-forces the
    quantiser indices (for decoder parity under bf16 code flips, SURVEY F9)."""
    BT, _, H, W = x.shape
    t = arch.tf
    b = BT // t
    inter = {}
    mean = torch.tensor(IMAGENET_MEAN, dtype=x.dtype).view(1, 3, 1, 1)
    std = torch.tensor(IMAGENET_STD, dtype=x.dtype).view(1, 3, 1, 1)
    cond = bisenet(sd, 'conditionnet', (x - mean) / std)                       # :606-607
    cond = conv(sd, 'convpos', cond)                                           # :609
    th, tw = cond.shape[2:]
    tc = cond.shape[1]
    pos = cond.view(b, t, tc, th, tw).permute(0, 2, 1, 3, 4).reshape(b, tc, t * th * tw).permute(2, 0, 1)
    h, feats = encoder_forward(sd, arch, x)                                    # :626
    lq = conv(sd, 'quant_conv', h)                                             # :631-633
    fe = linear(sd, 'feat_emb', lq.flatten(2).permute(2, 0, 1))                # :638  [hw, b*t, E]
    cc = fe.shape[-1]
    q = fe.view(th * tw, b, t, cc).permute(2, 0, 1, 3).reshape(t * th * tw, b, cc)   # frame-major
    inter['query_in'] = q
    inter['pos'] = pos
    for i in range(arch.n_layers):
        q = transformer_sa_layer(sd, 'ft_layers.%d' % i, q, pos, arch.n_head)  # :642-643
    inter['query_out'] = q
    qo = q.view(t, th * tw, b, cc).permute(1, 2, 0, 3).reshape(th * tw, b * t, cc)
    logits = F.linear(layer_norm(sd, 'idx_pred_layer.0', qo), sd['idx_pred_layer.1.weight'])
    logits = logits.transpose(0, 1).reshape(b * t, th, tw, 1, -1)              # :646-649
    lq_nhwc = lq.permute(0, 2, 3, 1)
    if code_only:
        return logits, lq_nhwc
    codes = logits.argmax(-1) if force_codes is None else force_codes          # :663
    quant = embed_code(sd['quantizer.codebooks.0.weight'], codes).permute(0, 3, 1, 2).contiguous()
    if adain_on:
        quant = adain(quant, lq)                                               # :670-671
    z = conv(sd, 'post_quant_conv', quant)
    inter['z'] = z
    out = decoder_forward(sd, arch, z, feats, w)
    if return_intermediates:
        inter.update(cond=cond, enc_feats=feats, enc_h=h, codes=codes)
        return (out, logits, lq_nhwc), inter
    return out, logits, lq_nhwc


def tdcrqvae3_forward(sd, arch, x, code_only=False):
    """TDCRQVAE3.forward (`archs/tdcrqvae3_arch.py:760-783`, RQBottleneck :294-338) for depth 1:
    encode -> L2 argmin -> embed -> decode.  Returns (out, commitment_loss, codes [b*3,h,w,1])."""
    h, _ = encoder_forward(sd, arch, x)
    z_e = conv(sd, 'quant_conv', h).permute(0, 2, 3, 1).contiguous()
    cb = sd['quantizer.codebooks.0.weight']
    codes = l2_argmin(cb, z_e).unsqueeze(-1)
    z_q = embed_code(cb, codes)
    loss = (z_e - z_q).pow(2.0).mean()
    if code_only:
        return z_q, loss, codes
    out = decoder_forward(sd, arch, conv(sd, 'post_quant_conv', z_q.permute(0, 3, 1, 2).contiguous()))
    return out, loss, codes
