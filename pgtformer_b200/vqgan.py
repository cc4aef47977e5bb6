"""H100 launch sequences of VQAutoEncoder (`archs/vqgan_arch.py:344-411`) and CodeFormer (`archs/codeformer_arch.py:
229-366`) over libpgt_b200.so.

Both walk the flat `encoder.blocks` / `generator.blocks` lists of spec.VQGANArch, as the reference's forward does, on the
blocks Engine already has: ResBlock is td_resblock with the `conv_out` shortcut, AttnBlock is attn_block, Downsample the
stride-2 conv, Upsample up2x, the transformer global_transformer and the SFT fusion sft_tail.  Layout as in engine.py:
channels-last bf16 feature maps [b, H, W, C]; the latent's token rows are in (image, y, x) order, which is the
reference's b(hw) order of logits and codes.  Every op is a call into the C ABI; there is no PyTorch / CPU fallback."""
import torch

from . import ops
from .engine import BF, Engine, _on_device, _pack_conv, _pack_lin, _pack_rgb, _pack_up2x
from .spec import VQGANArch

F32 = torch.float32


class VQGANEngine(Engine):
    codeformer = False

    def arch_class(self, g):
        return VQGANArch(g, self.codeformer)

    def _repack(self):
        """Kernel layouts by the spec's block kinds (an Upsample conv is `generator.blocks.N.conv`, a Downsample conv
        `encoder.blocks.N.conv`: no name pattern tells them apart)."""
        sd, w = self._sd, self.w
        for name, t in sd.items():
            if t.dtype.is_floating_point and t.dim() == 1:
                w[name] = t.float().contiguous()
            elif name.endswith('.weight') and t.dim() == 4:
                w[name] = _pack_conv(t.float()) if t.shape[2] == 3 else _pack_lin(t.float())
            elif name.endswith('.weight') and t.dim() == 2 and name != 'quantize.embedding.weight':
                w[name] = _pack_lin(t.float())
        for prefix, blocks in (('encoder', self.arch.enc_blocks), ('generator', self.arch.gen_blocks)):
            for i, (kind, *_rest) in enumerate(blocks):
                p = '%s.blocks.%d' % (prefix, i)
                if kind == 'up':
                    w[p + '.conv.weight'] = _pack_up2x(sd[p + '.conv.weight'].float())
                elif kind == 'conv_in' and prefix == 'encoder':
                    w[p + '.weight'] = _pack_rgb(sd[p + '.weight'].float())
        w['codebook'] = self._f32('quantize.embedding.weight')
        self._repack_attn_qkv()

    def _stats_tiles(self, H, W, cout, ksize, stride, pad_lo):
        """Fused statistics only where the conv's tile grid divides the frame: VQAutoEncoder takes any multiple of 128,
        and at, say, 256 x 384 the 256-channel levels (48 and 24 columns) get 32- and 16-column tiles, whose last
        column of tiles would add rows past the frame's edge to the statistics (pgt_conv_tiles_exact)."""
        return ops.conv_tiles_exact(H, W, cout, ksize, stride, pad_lo)

    def _codebook_pack(self, d=0):
        if 'codebook.pack' not in self.w:
            self.w['codebook.pack'] = ops.codebook_pack(self.w['codebook'], self.arch.n_embed)
        return self.w['codebook.pack']

    # ------------------------------------------------------------------ encoder / generator
    def _walk(self, prefix, blocks, h, lo, hi, taps=None):
        """Runs blocks[lo:hi] of `prefix` on h; with taps (flat index -> key) returns {key: output after that block}."""
        feats = {}
        for i in range(lo, hi):
            kind, cin, cout, _ = blocks[i]
            p = '%s.blocks.%d' % (prefix, i)
            # the next block reads this output through a GroupNorm: its statistics come from this block's epilogue
            nxt = blocks[i + 1][0] in ('res', 'attn', 'norm') if i + 1 < len(blocks) else False
            if kind == 'res':
                h = self.td_resblock(h, p, cout, gn_next=nxt, shortcut='conv_out')
            elif kind == 'attn':
                h = self.attn_block(h, p, gn_next=nxt)
            elif kind == 'down':
                h = self._conv3(h, p + '.conv', cout, stride=2, pad_lo=0, gn_out=True)
            elif kind == 'up':
                h = self.up2x(h, p + '.conv')
            else:
                raise AssertionError(kind)
            if taps is not None and i in taps:
                feats[taps[i]] = h
        return h, feats

    def encoder(self, x, taps=None):
        """encoder.blocks[:-2] on x fp32 NCHW [b,3,H,W] -> (h bf16 [b,h,w,C] with the final GroupNorm's statistics,
        {key: tapped block output})."""
        a = self.arch
        h = self.conv_in(x, 'encoder.blocks.0')
        return self._walk('encoder', a.enc_blocks, h, 1, len(a.enc_blocks) - 2, taps)

    def encoder_out(self, h, out, nchw=False):
        """The encoder tail: GroupNorm (no SiLU) -> conv 3x3 to emb_dim, into out (fp32 NHWC rows, fp32 NCHW with
        nchw, or bf16 NHWC).  The GroupNorm runs on its own pass: the fused conv_gn kernel always applies SiLU."""
        n = len(self.arch.enc_blocks)
        y = getattr(h, '_pgt_normed', None)
        if y is None:
            y = self._gn(h, 'encoder.blocks.%d' % (n - 2), silu=False)
            h._pgt_normed = y
        return self._conv3(y, 'encoder.blocks.%d' % (n - 1), self.arch.embed_dim, out=out, nchw=nchw)

    def generator(self, z, feats=None, wgt=0.0):
        """generator.blocks on z bf16 [b,h,w,emb_dim] -> fp32 NCHW [b,3,H,W]; with feats and wgt > 0 CodeFormer's
        Fuse_sft_block after the blocks of arch.fuse_gen (`archs/codeformer_arch.py:356-363`)."""
        a = self.arch
        blocks = a.gen_blocks
        h = self._conv3(z, 'generator.blocks.0', blocks[0][2], gn_out=True)
        fuse = a.fuse_gen if (feats is not None and wgt > 0) else {}
        i = 1
        for j in sorted(fuse) + [len(blocks) - 2]:
            h, _ = self._walk('generator', blocks, h, i, j + 1 if j in fuse else j)
            if j in fuse:
                h = self.fuse(feats[fuse[j]], h, fuse[j], wgt)
            i = j + 1
        n = len(blocks)
        return self.decoder_out(h, 'generator.blocks.%d' % (n - 2), 'generator.blocks.%d' % (n - 1), silu=False, out_ch=3)

    def fuse(self, enc, dec, key, wgt):
        """Fuse_sft_block (`archs/codeformer_arch.py:218-226`): the concat [enc | dec] -> sft_tail; the output feeds
        the next ResBlock's GroupNorm."""
        Fr, H, W, C = dec.shape
        cat = self._new(Fr, H, W, 2 * C)
        ops.copy2d(enc, cat[..., :C])
        ops.copy2d(dec, cat[..., C:])
        return self.sft_tail(cat, dec, 'fuse_convs_dict.' + key, wgt, gn_next=True)

    # ------------------------------------------------------------------ VQAutoEncoder.forward
    def _check(self, x):
        a = self.arch
        x = x.to(self.dev, F32).contiguous()
        b, c, H, W = x.shape
        m = 4 * a.down
        if c != 3 or b == 0 or H == 0 or W == 0 or H % m or W % m:
            raise ValueError('expected images [b, 3, H, W] with H, W multiples of %d, got %s' % (m, tuple(x.shape)))
        return x

    @_on_device
    @torch.no_grad()
    def encode(self, x):
        """Encoder.forward (`archs/vqgan_arch.py:285-289`): x [b,3,H,W] -> z fp32 NHWC [b, H/32, W/32, emb_dim]."""
        a = self.arch
        x = self._check(x)
        b, _, H, W = x.shape
        h, _ = self.encoder(x)
        z = self._new(b, H // a.down, W // a.down, a.embed_dim, dtype=F32)
        return self.encoder_out(h, z)

    @_on_device
    @torch.no_grad()
    def forward(self, x, code_only=False, usage=None, force_codes=None):
        """VQAutoEncoder.forward (`archs/vqgan_arch.py:405-411`): (out fp32 [b,3,H,W] or, code_only, quant fp32 NCHW
        [b, emb_dim, h, w], codebook_loss, quant_stats) with VectorQuantizer.forward's statistics (`:42-84`); usage
        (int32 [K], the module's buffer) receives the code counts.  force_codes (int64 [b*h*w], decoder parity checks)
        replaces the argmin codes, statistics included."""
        a = self.arch
        z = self.encode(x)
        b, hh, ww, E = z.shape
        T, K = b * hh * ww, a.n_embed
        codes = torch.empty(T, dtype=torch.int64, device=self.dev)
        zr = z.view(T, E)
        ops.l2_argmin_tc(zr, self.w['codebook'], self._codebook_pack(), K, codes)
        if force_codes is not None:
            codes = force_codes.to(self.dev, torch.int64).reshape(T).contiguous()
        scalars = self._new(3, dtype=F32)
        min_enc = self._new(T, K, dtype=F32)
        scores = self._new(T, dtype=F32)
        zq = self._new(b, E, hh, ww, dtype=F32) if code_only else None
        zq16 = None if code_only else self._new(b, hh, ww, E)
        ops.vq_stats(zr, self.w['codebook'], codes, hh * ww, a.beta, scalars, zq_nchw=zq, zq_bf16=zq16, min_enc=min_enc,
                     scores=scores, usage=usage)
        stats = {'perplexity': scalars[1], 'min_encodings': min_enc, 'min_encoding_indices': codes.view(T, 1),
                 'min_encoding_scores': scores.view(T, 1), 'mean_distance': scalars[2]}
        self.last_z = z
        if code_only:
            return zq, scalars[0], stats
        return self.generator(zq16), scalars[0], stats


class CodeFormerEngine(VQGANEngine):
    codeformer = True

    def _repack(self):
        super()._repack()
        sd, w = self._sd, self.w
        E = self.arch.dim_embd
        for i in range(self.arch.n_layers):
            p = 'ft_layers.%d.self_attn' % i
            wi, bi = sd[p + '.in_proj_weight'].float(), sd[p + '.in_proj_bias'].float()
            w[p + '.qk.weight'], w[p + '.qk.bias'] = _pack_lin(wi[:2 * E]), bi[:2 * E].contiguous()
            w[p + '.v.weight'], w[p + '.v.bias'] = _pack_lin(wi[2 * E:]), bi[2 * E:].contiguous()
        w['position_emb'] = sd['position_emb'].to(BF).contiguous()
        self._pos = {}

    def pos(self, b):
        """position_emb tiled over the batch: [b * L, dim_embd] bf16, built once per batch size."""
        if b not in self._pos:
            self._pos[b] = self.w['position_emb'].repeat(b, 1).contiguous()
        return self._pos[b]

    @_on_device
    @torch.no_grad()
    def forward(self, x, w=0.0, adain=False, code_only=False, force_codes=None):
        """CodeFormer.forward (`archs/codeformer_arch.py:303-366`) on x [b,3,512,512]: (out fp32 NCHW, logits fp32
        [b, 256, K], lq_feat fp32 NCHW [b, 256, 16, 16]), or (logits, lq_feat) with code_only.

        Codes are the first maximum of the fp32 logits (argmax_gather).  The reference takes topk(softmax(logits), 1):
        the same index except where two logits are close enough for their softmax probabilities to round to the same
        fp32 value, when it may return the later one.  force_codes (int64 [b, 256]) replaces the codes (teacher-forced
        decoder checks)."""
        a = self.arch
        x = self._check(x)
        b, _, H, W = x.shape
        if H != a.img_size or W != a.img_size:
            raise ValueError('CodeFormer runs %d^2 images only, got %s' % (a.img_size, tuple(x.shape)))
        hh, ww = H // a.down, W // a.down
        L, E = hh * ww, a.embed_dim
        T = b * L
        fusing = (not code_only) and float(w) > 0
        h, feats = self.encoder(x, a.fuse_enc if fusing else None)
        lq_nchw = self.encoder_out(h, self._new(b, E, hh, ww, dtype=F32), nchw=True)
        lq = self.encoder_out(h, self._new(b, hh, ww, E))
        logits = self.global_transformer(lq.view(T, E), self.pos(b), b)
        if code_only:
            return logits.view(b, L, a.n_embed), lq_nchw
        codes = torch.empty(T, dtype=torch.int64, device=self.dev)
        idx_in = force_codes.to(self.dev, torch.int64).reshape(T).contiguous() if force_codes is not None else None
        if adain:
            quant = self._new(T, E, dtype=F32)
            ops.argmax_gather(logits, self.w['codebook'], codes, quant, idx_in=idx_in)
            quant = ops.adain(quant.view(b, L, E), lq.view(b, L, E), self._new(b, L, E))
        else:
            quant = self._new(T, E)
            ops.argmax_gather(logits, self.w['codebook'], codes, quant, idx_in=idx_in)
        self.last_codes = (codes if idx_in is None else idx_in).view(b, L)
        out = self.generator(quant.view(b, hh, ww, E), feats, float(w))
        return out, logits.view(b, L, a.n_embed), lq_nchw
