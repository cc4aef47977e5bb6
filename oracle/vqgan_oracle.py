"""TEST INFRASTRUCTURE ONLY — CPU restatement of the reference's VQAutoEncoder (`archs/vqgan_arch.py:14-414`) and
CodeFormer (`archs/codeformer_arch.py:229-366`), functional on a state dict and the block list of
pgtformer_b200.spec.VQGANArch.  Only tests/ import it; it is pinned against the outputs of the reference's own modules
(tests/golden/codeformer_*.pt / vqgan_*.pt, minted by `python -m oracle.make_codeformer_golden`).

Reused where the math is identical: Downsample / Upsample (`vqgan_arch.py:131-152`) are pgt_oracle's, AttnBlock
(`:181-240`) is tdrqvae_oracle's, TransformerSALayer (`codeformer_arch.py:102-137`) and AdaIN (`:15-46`) pgt_oracle's."""
import torch
import torch.nn.functional as F

from oracle.pgt_oracle import adain, conv, downsample, group_norm, layer_norm, silu, transformer_sa_layer, upsample
from oracle.tdrqvae_oracle import attn_block


def res_block(sd, p, x):
    """ResBlock.forward (`archs/vqgan_arch.py:167-178`): GN -> swish -> conv3x3, twice, + x (1x1 conv_out of x when the
    width changes)."""
    h = conv(sd, p + '.conv1', silu(group_norm(sd, p + '.norm1', x)), padding=1)
    h = conv(sd, p + '.conv2', silu(group_norm(sd, p + '.norm2', h)), padding=1)
    if (p + '.conv_out.weight') in sd:
        x = conv(sd, p + '.conv_out', x)
    return h + x


def block(sd, b, x):
    """One entry of Encoder.blocks / Generator.blocks (`archs/vqgan_arch.py:252-341`), a spec.Block."""
    p, kind = b.prefix, b.kind
    if kind in ('conv_in', 'conv_out'):
        return conv(sd, p, x, padding=1)
    if kind == 'res':
        return res_block(sd, p, x)
    if kind == 'attn':
        return attn_block(sd, p, x)
    if kind == 'down':
        return downsample(sd, p, x)
    if kind == 'up':
        return upsample(sd, p, x)
    return group_norm(sd, p, x)                           # normalize(); last_silu=False adds no SiLU (:279-282)


def encoder(sd, arch, x, taps=None):
    """Encoder.forward (`:285-289`); returns (z NCHW, {taps[i]: output of block i})."""
    feats = {}
    for i, b in enumerate(arch.enc_blocks):
        x = block(sd, b, x)
        if taps and i in taps:
            feats[taps[i]] = x.clone()
    return x, feats


def generator(sd, arch, x, fuse=None):
    """Generator.forward (`:337-341`); fuse(b, x) -> x at each `fuse` block b (CodeFormer's SFT fusion)."""
    for b in arch.dec_blocks:
        if b.kind != 'fuse':
            x = block(sd, b, x)
        elif fuse is not None:
            x = fuse(b, x)
    return x


def vector_quantize(sd, z, beta):
    """VectorQuantizer.forward (`archs/vqgan_arch.py:42-84`) in eval mode: (z_q NCHW, loss, stats, counts [K])."""
    emb = sd['quantize.embedding.weight']
    zp = z.permute(0, 2, 3, 1).contiguous()
    zf = zp.view(-1, emb.shape[1])
    d = (zf ** 2).sum(dim=1, keepdim=True) + (emb ** 2).sum(1) - 2 * torch.matmul(zf, emb.t())
    mean_distance = torch.mean(d)
    scores, idx = torch.topk(d, 1, dim=1, largest=False)
    scores = torch.exp(-scores / 10)
    min_enc = torch.zeros(idx.shape[0], emb.shape[0]).to(zp)
    min_enc.scatter_(1, idx, 1)
    counts = torch.bincount(idx.view(-1), minlength=emb.shape[0]).to(torch.int32)
    z_q = torch.matmul(min_enc, emb).view(zp.shape)
    loss = torch.mean((z_q - zp) ** 2) + beta * torch.mean((z_q - zp) ** 2)
    z_q = zp + (z_q - zp)
    e_mean = torch.mean(min_enc, dim=0)
    perplexity = torch.exp(-torch.sum(e_mean * torch.log(e_mean + 1e-10)))
    stats = {'perplexity': perplexity, 'min_encodings': min_enc, 'min_encoding_indices': idx,
             'min_encoding_scores': scores, 'mean_distance': mean_distance}
    return z_q.permute(0, 3, 1, 2).contiguous(), loss, stats, counts


def vqgan_forward(sd, arch, x, code_only=False):
    """VQAutoEncoder.forward (`:405-411`): (out or quant, codebook_loss, quant_stats, counts); also z."""
    z, _ = encoder(sd, arch, x)
    quant, loss, stats, counts = vector_quantize(sd, z, arch.beta)
    res = quant if code_only else generator(sd, arch, quant)
    return res, loss, stats, counts, z


def fuse_sft(sd, p, enc, dec, w):
    """Fuse_sft_block.forward (`archs/codeformer_arch.py:218-226`)."""
    e = res_block(sd, p + '.encode_enc', torch.cat([enc, dec], dim=1))
    scale = conv(sd, p + '.scale.2', F.leaky_relu(conv(sd, p + '.scale.0', e, padding=1), 0.2), padding=1)
    shift = conv(sd, p + '.shift.2', F.leaky_relu(conv(sd, p + '.shift.0', e, padding=1), 0.2), padding=1)
    return dec + w * (dec * scale + shift)


def codeformer_forward(sd, arch, x, w=0.0, adain_on=False, code_only=False, force_codes=None):
    """CodeFormer.forward (`archs/codeformer_arch.py:303-366`): (out, logits [b, hw, K], lq_feat NCHW), or
    (logits, lq_feat) with code_only.  Codes are topk(softmax(logits), 1) as in the reference; force_codes [b, hw]
    replaces them."""
    lq, feats = encoder(sd, arch, x, taps=arch.enc_taps)
    b = lq.shape[0]
    pos = sd['position_emb'].unsqueeze(1).repeat(1, b, 1)
    q = F.linear(lq.flatten(2).permute(2, 0, 1), sd['feat_emb.weight'], sd['feat_emb.bias'])
    for i in range(arch.n_layers):
        q = transformer_sa_layer(sd, 'ft_layers.%d' % i, q, pos, heads=arch.n_head)
    logits = F.linear(layer_norm(sd, 'idx_pred_layer.0', q), sd['idx_pred_layer.1.weight']).permute(1, 0, 2)
    if code_only:
        return logits, lq
    if force_codes is None:
        _, top_idx = torch.topk(F.softmax(logits, dim=2), 1, dim=2)
    else:
        top_idx = force_codes.reshape(b, -1, 1)
    emb = sd['quantize.embedding.weight']
    hh, ww = lq.shape[2], lq.shape[3]
    quant = F.embedding(top_idx.reshape(-1), emb).view(b, hh, ww, -1).permute(0, 3, 1, 2).contiguous()
    if adain_on:
        quant = adain(quant, lq)

    def fuse(b, h):
        return fuse_sft(sd, b.prefix, feats[b.src], h, w) if w > 0 else h
    return generator(sd, arch, quant, fuse), logits, lq
