"""TEST INFRASTRUCTURE ONLY — CPU restatement of the reference's TDRQVAE (`archs/tdrqvae_arch.py:787-976`), functional
on a state dict.  Only tests/ import it; it is pinned against the outputs of the reference's own module
(tests/golden/tdrqvae_*.pt, minted by `python -m oracle.make_tdrqvae_golden`).

Reused where the math is identical: ResnetBlock (`:121-141`) is pgt_oracle.td_resblock (GN -> SiLU -> conv3x3, twice,
+ 1x1 nin_shortcut), Downsample / Upsample are pgt_oracle's, the Video-Swin BasicLayer is swin3d_oracle.basic_layer and
the quantiser (L2 argmin over the rows before the padding row, embed, soft codes) is pgt_oracle / codec_oracle's.
Restated here: AttnBlock (`:179-203`), Encoder / Decoder.forward (`:650-680`, `:753-784`) and the model methods."""
import torch
import torch.nn.functional as F

from oracle.codec_oracle import soft_codes
from oracle.pgt_oracle import conv, downsample, embed_code, group_norm, l2_argmin, silu, td_resblock, upsample
from oracle.swin3d_oracle import basic_layer


def attn_block(sd, p, x):
    """AttnBlock.forward: GroupNorm (no SiLU), 1x1 q / k / v, softmax(q k^T * C^-1/2) v over the H*W tokens of each
    frame, proj_out, + x.  x [F, C, H, W]."""
    h = group_norm(sd, p + '.norm', x)
    q, k, v = (conv(sd, '%s.%s' % (p, n), h) for n in 'qkv')
    b, c, hh, ww = q.shape
    q = q.reshape(b, c, hh * ww).permute(0, 2, 1)
    w_ = torch.bmm(q, k.reshape(b, c, hh * ww)) * (int(c) ** (-0.5))
    w_ = F.softmax(w_, dim=2)
    h = torch.bmm(v.reshape(b, c, hh * ww), w_.permute(0, 2, 1)).reshape(b, c, hh, ww)
    return x + conv(sd, p + '.proj_out', h)


def encoder_forward(sd, arch, x):
    h = conv(sd, 'encoder.conv_in', x, padding=1)
    for lvl in range(arch.num_levels):
        for b in range(arch.num_res_blocks):
            h = td_resblock(sd, 'encoder.down.%d.block.%d' % (lvl, b), h)
            if arch.level_has_attn[lvl]:
                h = attn_block(sd, 'encoder.down.%d.attn.%d' % (lvl, b), h)
        if lvl != arch.num_levels - 1:
            h = downsample(sd, 'encoder.down.%d.downsample' % lvl, h)
    h = td_resblock(sd, 'encoder.mid.block_1', h)
    h = attn_block(sd, 'encoder.mid.attn_1', h)
    h = td_resblock(sd, 'encoder.mid.block_2', h)
    return conv(sd, 'encoder.conv_out', silu(group_norm(sd, 'encoder.norm_out', h)), padding=1)


def decoder_forward(sd, arch, z):
    h = conv(sd, 'decoder.conv_in', z, padding=1)
    h = td_resblock(sd, 'decoder.mid.block_1', h)
    h = attn_block(sd, 'decoder.mid.attn_1', h)
    h = td_resblock(sd, 'decoder.mid.block_2', h)
    for lvl in reversed(range(arch.num_levels)):
        for b in range(arch.num_res_blocks + 1):
            h = td_resblock(sd, 'decoder.up.%d.block.%d' % (lvl, b), h)
            if arch.level_has_attn[lvl]:
                h = attn_block(sd, 'decoder.up.%d.attn.%d' % (lvl, b), h)
        if lvl != 0:
            h = upsample(sd, 'decoder.up.%d.upsample' % lvl, h)
    return conv(sd, 'decoder.conv_out', silu(group_norm(sd, 'decoder.norm_out', h)), padding=1)


def encode(sd, arch, x):
    """TDRQVAE.encode (`:863-866`): frames [F,3,H,W] -> NHWC z_e [F, H/16, W/16, E]."""
    return conv(sd, 'quant_conv', encoder_forward(sd, arch, x)).permute(0, 2, 3, 1).contiguous()


def decode(sd, arch, z_q):
    """TDRQVAE.decode (`:868-872`): NHWC z_q -> post_quant_conv -> Decoder."""
    return decoder_forward(sd, arch, conv(sd, 'post_quant_conv', z_q.permute(0, 3, 1, 2).contiguous()))


def tdswin(sd, arch, name, z, b, t):
    """tdswin_pre / tdswin_post on NHWC latents [b*t, h, w, E] (`:849-850`, `:853-854`) -> same shape."""
    _, hh, ww, E = z.shape
    x = z.view(b, t, hh, ww, E).permute(0, 4, 1, 2, 3)
    y = basic_layer(sd, name, x, arch.stages_atten, arch.num_head, arch.window_size)
    return y.permute(0, 2, 3, 4, 1).reshape(b * t, hh, ww, E)


def forward(sd, arch, x, code_only=False, force_codes=None, return_latents=False):
    """TDRQVAE.forward (`:843-861`) for depth 1 on x [b,t,3,H,W]: (out [b,t,3,H,W] or, code_only, z_q after
    tdswin_post [b,t,h,w,E], quant_loss, code [b,t,h,w,1]).  force_codes [b*t,h,w,1] replaces the argmin codes before
    tdswin_post.  With return_latents also {'z_e', 'z_pre', 'dist'} (the L2 distances of z_pre to every code)."""
    b, t, c, H, W = x.shape
    z_e = encode(sd, arch, x.reshape(b * t, c, H, W))
    z = tdswin(sd, arch, 'tdswin_pre', z_e, b, t)
    cb = sd['quantizer.codebooks.0.weight']
    code = l2_argmin(cb, z).unsqueeze(-1)
    q = embed_code(cb, code)
    loss = (z - q).pow(2.0).mean()
    q = z + (q - z) if force_codes is None else embed_code(cb, force_codes)     # RQBottleneck.forward (:460-461)
    z_q = tdswin(sd, arch, 'tdswin_post', q, b, t)
    _, hh, ww, E = z.shape
    res = z_q.view(b, t, hh, ww, E) if code_only else decode(sd, arch, z_q).view(b, t, c, H, W)
    res = (res, loss, code.view(b, t, hh, ww, 1))
    if return_latents:
        from oracle.pgt_oracle import l2_distances
        return res, {'z_e': z_e, 'z_pre': z, 'dist': l2_distances(cb, z)}
    return res


def decode_code(sd, arch, code):
    """TDRQVAE.decode_code (`:912-917`): codebook rows of [F,h,w,1] codes, decoded without tdswin_post."""
    return decode(sd, arch, embed_code(sd['quantizer.codebooks.0.weight'], code))


def get_soft_codes(sd, arch, xs, temp=1.0):
    """TDRQVAE.get_soft_codes (`:904-910`), stochastic=False: on encode(xs), without tdswin_pre."""
    return soft_codes(sd['quantizer.codebooks.0.weight'], encode(sd, arch, xs), temp)
