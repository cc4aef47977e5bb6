"""H100 launch sequences of VQAutoEncoder (`archs/vqgan_arch.py:344-411`) and CodeFormer (`archs/codeformer_arch.py:
229-366`) over libpgt_b200.so.

Both walk the flat `encoder.blocks` / `generator.blocks` lists of spec.VQGANArch, as the reference's forward does, on the
blocks Engine already has: ResBlock is td_resblock with the `conv_out` shortcut, AttnBlock is attn_block, Downsample the
stride-2 conv, Upsample up2x, the generator Engine.decoder, the transformer global_transformer and the SFT fusion
sft_tail.  Layout as in engine.py: channels-last bf16 feature maps [b, H, W, C]; the latent's token rows are in
(image, y, x) order, which is the reference's b(hw) order of logits and codes.  Every op is a call into the C ABI; there
is no PyTorch / CPU fallback."""
import torch

from . import ops
from .engine import Engine, _on_device
from .spec import VQGANArch

F32 = torch.float32


class VQGANEngine(Engine):
    codeformer = False

    def arch_class(self, g):
        return VQGANArch(g, self.codeformer)

    # ------------------------------------------------------------------ encoder
    def encoder(self, x, taps=None):
        """encoder.blocks[:-2] on x fp32 NCHW [b,3,H,W] -> (h bf16 [b,h,w,C] with the final GroupNorm's statistics,
        {key: tapped block output})."""
        blocks = self.arch.enc_blocks
        return self._walk(blocks, x, 0, len(blocks) - 2, taps)

    def encoder_out(self, h, out, nchw=False):
        """The encoder tail: GroupNorm (no SiLU) -> conv 3x3 to emb_dim, into out (fp32 NHWC rows, fp32 NCHW with
        nchw, or bf16 NHWC).  The GroupNorm runs on its own pass."""
        norm, conv = self.arch.enc_blocks[-2:]
        y = getattr(h, '_pgt_normed', None)
        if y is None:
            y = self._gn(h, norm.prefix, silu=False)
            h._pgt_normed = y
        return self._conv3(y, conv.prefix, conv.cout, out=out, nchw=nchw)

    def fuse_sft(self, enc, dec, key, wgt, gn_next=False):
        """Fuse_sft_block (`archs/codeformer_arch.py:218-226`): the concat [enc | dec] -> sft_tail."""
        Fr, H, W, C = dec.shape
        cat = self._new(Fr, H, W, 2 * C)
        ops.copy2d(enc, cat[..., :C])
        ops.copy2d(dec, cat[..., C:])
        return self.sft_tail(cat, dec, 'fuse_convs_dict.' + key, wgt, gn_next)

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
        self._argmin(zr, self.w['codebook'], self._codebook_pack(), self._n_embed(0), codes)
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
        return self.decoder(zq16), scalars[0], stats

    def counted_forward(self, x, usage, code_only=False):
        """forward with the usage buffer as a positional tensor argument (the form Engine.graphed replays)."""
        return self.forward(x, code_only=code_only, usage=usage)


class CodeFormerEngine(VQGANEngine):
    codeformer = True

    def pos(self, b):
        """position_emb tiled over the batch: [b * L, dim_embd] bf16, built once per batch size."""
        key = 'position_emb.%d' % b
        if key not in self.w:
            self.w[key] = self.w['position_emb'].repeat(b, 1).contiguous()
        return self.w[key]

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
        h, feats = self.encoder(x, a.enc_taps if fusing else None)
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
        out = self.decoder(quant.view(b, hh, ww, E), feats, float(w))
        return out, logits.view(b, L, a.n_embed), lq_nchw
